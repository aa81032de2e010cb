"""lizard_b200 -- thin ctypes binding over liblizard_b200.so (the C-ABI in include/lizard_b200.h).

The product is the shared library: hand-written sm_90a CUDA kernels behind Lizard's own C API
(`Lizard_compress`, `Lizard_decompress_safe`, ...) plus batch entry points.  This module only exists so
the tests and bench.py (Python) can call that C-ABI; it contains no codec logic and there is NO fallback:
if the library is missing, or no H100 is present, calls raise.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LIZARDB200_LIB") or os.path.join(_HERE, "liblizard_b200.so")     # the override is for A/B builds (tools/)
DATAGEN_PATH = os.path.join(os.path.dirname(_HERE), "tools", "libdatagen.so")   # bench / test input generator, not product code

BLOCK_SIZE = 1 << 17
_lib = None
_dg = None


class LizardB200Error(RuntimeError):
    pass


def lib():
    """Load liblizard_b200.so (built by __graft_entry__.build()); raises if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LizardB200Error(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        c_int_p = ctypes.POINTER(ctypes.c_int)
        vpp = ctypes.POINTER(ctypes.c_void_p)
        L.Lizard_versionNumber.restype = ctypes.c_int
        L.Lizard_compressBound.argtypes = [ctypes.c_int]
        L.Lizard_sizeofState.argtypes = [ctypes.c_int]
        L.Lizard_compress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.Lizard_compress_extState.argtypes = [ctypes.c_void_p] + L.Lizard_compress.argtypes
        L.Lizard_decompress_safe.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.LizardB200_lastError.restype = ctypes.c_char_p
        L.LizardB200_createDecompressionStream.argtypes = [ctypes.POINTER(ctypes.c_void_p)]
        L.LizardB200_freeDecompressionStream.argtypes = [ctypes.c_void_p]
        L.LizardB200_decompressStream.restype = ctypes.c_size_t
        L.LizardB200_decompressStream.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t),
                                                  ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p]
        L.LizardB200_launchCount.restype = ctypes.c_ulonglong
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        L.LizardB200_createCompressionStream.argtypes = [ctypes.POINTER(vp)]
        L.LizardB200_freeCompressionStream.argtypes = [vp]
        L.LizardB200_compressStreamBegin.argtypes = [vp, vp, sz, vp, vp, vp]
        L.LizardB200_compressStreamUpdate.argtypes = [vp, vp, sz, vp, sz, vp, vp]
        L.LizardB200_compressStreamFlush.argtypes = [vp, vp, sz, vp, vp]
        L.LizardB200_compressStreamEnd.argtypes = [vp, vp, sz, vp, vp]
        for f in ("Begin", "Update", "Flush", "End"):
            getattr(L, "LizardB200_compressStream" + f).restype = sz
        L.LizardB200_compress_batch.argtypes = [vpp, c_int_p, vpp, c_int_p, c_int_p, ctypes.c_int, ctypes.c_int]
        L.LizardB200_decompress_batch.argtypes = [vpp, c_int_p, vpp, c_int_p, c_int_p, ctypes.c_int]
        L.Lizard_decompress_safe_partial.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.LizardB200_decompress_partial_batch.argtypes = [vpp, c_int_p, vpp, c_int_p, c_int_p, c_int_p, ctypes.c_int]
        L.Lizard_decompress_safe_usingDict.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                       ctypes.c_void_p, ctypes.c_int]
        L.Lizard_createStreamDecode.restype = ctypes.c_void_p
        L.Lizard_freeStreamDecode.argtypes = [ctypes.c_void_p]
        L.Lizard_setStreamDecode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.Lizard_decompress_safe_continue.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.LizardB200_decompress_dict_batch.argtypes = [vpp, c_int_p, vpp, c_int_p, vpp, c_int_p, c_int_p, ctypes.c_int]
        dev_args = [ctypes.c_void_p] * 7 + [ctypes.c_uint]
        L.LizardB200_decompress_device.argtypes = dev_args + [ctypes.c_void_p]
        L.LizardB200_decompress_partial_device.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_uint, ctypes.c_void_p]
        L.LizardB200_decompress_dict_device.argtypes = [ctypes.c_void_p] * 10 + [ctypes.c_uint, ctypes.c_void_p]
        L.LizardB200_compress_device.argtypes = dev_args + [ctypes.c_int, ctypes.c_void_p]
        L.LizardB200_compress_dict_batch.argtypes = [vpp, c_int_p, vpp, c_int_p, vpp, c_int_p, c_int_p, ctypes.c_int, ctypes.c_int]
        L.LizardB200_compress_dict_device.argtypes = [ctypes.c_void_p] * 10 + [ctypes.c_uint, ctypes.c_int, ctypes.c_void_p]
        L.Lizard_createStream.restype = ctypes.c_void_p
        L.Lizard_createStream.argtypes = [ctypes.c_int]
        L.Lizard_freeStream.argtypes = [ctypes.c_void_p]
        L.Lizard_loadDict.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.Lizard_compress_continue.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_int]
        L.Lizard_saveDict.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.LizardB200_gather_device.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_uint, ctypes.c_void_p]
        L.LizardB200_compress_blocks.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p,
                                                 ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.LizardB200_decompress_blocks.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                                   ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        u64p = ctypes.POINTER(ctypes.c_uint64)
        L.LizardB200_compressFrames.argtypes = [ctypes.c_void_p, u64p, u64p, ctypes.c_void_p, u64p, u64p,
                                                ctypes.POINTER(ctypes.c_size_t), ctypes.c_uint, ctypes.c_void_p, ctypes.c_void_p]
        L.LizardB200_decompressFrames.argtypes = [ctypes.c_void_p, u64p, u64p, ctypes.c_void_p, u64p, u64p,
                                                  ctypes.POINTER(ctypes.c_size_t), ctypes.c_uint, ctypes.c_void_p]
        L.LizardB200_decompressFramesAsync.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_uint, ctypes.c_uint, ctypes.c_size_t,
                                                                               ctypes.c_void_p]
        L.LizardB200_compressFramesAsync.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_uint, ctypes.c_void_p, ctypes.c_uint,
                                                     ctypes.c_size_t, ctypes.c_void_p]
        L.LizardF_isError.argtypes = [ctypes.c_size_t]
        L.LizardF_getErrorName.argtypes = [ctypes.c_size_t]
        L.LizardF_getErrorName.restype = ctypes.c_char_p
        _lib = L
    return _lib


def _check(status, what):
    if status != 0:
        raise LizardB200Error(f"{what} failed: status {status}: {lib().LizardB200_lastError().decode()}")


def compress_bound(n):
    return lib().Lizard_compressBound(n)


def compress(src: bytes, level: int, cap: int = None) -> bytes:
    """Lizard_compress on host bytes. Returns b'' when the library returns 0 (did not fit / failed)."""
    L = lib()
    cap = L.Lizard_compressBound(len(src)) if cap is None else cap
    dst = ctypes.create_string_buffer(max(cap, 1))
    n = L.Lizard_compress(src, dst, len(src), cap, level)
    return dst.raw[:n]


def decompress(src: bytes, max_size: int):
    """Lizard_decompress_safe on host bytes -> (return code, bytes)."""
    L = lib()
    dst = ctypes.create_string_buffer(max(max_size, 1))
    r = L.Lizard_decompress_safe(src, dst, len(src), max_size)
    return r, (dst.raw[:r] if r > 0 else b"")


def decompress_partial(src: bytes, target: int, max_size: int):
    """Lizard_decompress_safe_partial on host bytes -> (return code, bytes).  Decoding stops once `target` bytes are out;
    the return code may exceed the target (the reference's stopping rules, include/lizard_b200.h)."""
    L = lib()
    dst = ctypes.create_string_buffer(max(max_size, 1))
    r = L.Lizard_decompress_safe_partial(src, dst, len(src), target, max_size)
    return r, (dst.raw[:r] if r > 0 else b"")


def decompress_using_dict(src: bytes, dict: bytes, max_size: int, prefix: bool = False):
    """Lizard_decompress_safe_usingDict on host bytes -> (return code, bytes).  prefix=True lays the dictionary directly in
    front of the output buffer (the reference's in-place mode); otherwise it is an external dictionary."""
    L = lib()
    if prefix:
        buf = ctypes.create_string_buffer(bytes(dict), len(dict) + max(max_size, 1))
        dict_p, dst_p = ctypes.addressof(buf), ctypes.addressof(buf) + len(dict)
    else:
        d = ctypes.create_string_buffer(bytes(dict), max(len(dict), 1))
        buf = ctypes.create_string_buffer(max(max_size, 1))
        dict_p, dst_p = ctypes.addressof(d), ctypes.addressof(buf)
    r = L.Lizard_decompress_safe_usingDict(src, dst_p, len(src), max_size, dict_p, len(dict))
    out = ctypes.string_at(dst_p, r) if r > 0 else b""
    return r, out


def _batch(fn, units, caps, extra, targets=None, dicts=None):
    n = len(units)
    srcs = (ctypes.c_void_p * n)()
    sizes = (ctypes.c_int * n)()
    dsts = (ctypes.c_void_p * n)()
    dcaps = (ctypes.c_int * n)()
    res = (ctypes.c_int * n)()
    keep, outs = [], []
    for i, u in enumerate(units):
        b = ctypes.create_string_buffer(bytes(u), max(len(u), 1))
        keep.append(b)
        srcs[i] = ctypes.cast(b, ctypes.c_void_p)
        sizes[i] = len(u)
        o = ctypes.create_string_buffer(max(caps[i], 1))
        outs.append(o)
        dsts[i] = ctypes.cast(o, ctypes.c_void_p)
        dcaps[i] = caps[i]
    if targets is not None:
        st = fn(srcs, sizes, dsts, dcaps, (ctypes.c_int * n)(*targets), res, n, *extra)
    elif dicts is not None:
        st = fn(srcs, sizes, dsts, dcaps, dicts[0], dicts[1], res, n, *extra)
    else:
        st = fn(srcs, sizes, dsts, dcaps, res, n, *extra)
    _check(st, "batch call")
    return [(res[i], outs[i].raw[:res[i]] if res[i] > 0 else b"") for i in range(n)]


def compress_batch(units, level, caps=None):
    """LizardB200_compress_batch: list of bytes -> list of (result, compressed bytes)."""
    L = lib()
    caps = [L.Lizard_compressBound(len(u)) for u in units] if caps is None else caps
    return _batch(L.LizardB200_compress_batch, units, caps, (level,))


def _dict_args(dicts, n):
    """Per-unit dictionary pointers and sizes; units given the same bytes object share one buffer."""
    if len(dicts) != n:
        raise ValueError("one dictionary per unit")
    ptrs, sizes, held = (ctypes.c_void_p * n)(), (ctypes.c_int * n)(), {}
    for i, d in enumerate(dicts):
        if d:
            if id(d) not in held:
                held[id(d)] = ctypes.create_string_buffer(bytes(d), len(d))
            ptrs[i] = ctypes.addressof(held[id(d)])
            sizes[i] = len(d)
    return ptrs, sizes, held


def compress_dict_batch(units, dicts, level, caps=None):
    """LizardB200_compress_dict_batch: list of bytes, per-unit dictionary (bytes; b"" or None for none) -> list of (result,
    compressed bytes), each as Lizard_loadDict + Lizard_compress_continue with an external dictionary.  Units given the same
    bytes object share one dictionary buffer.  Levels 13-17, 21, 22, 34-38, 41 and 42."""
    L = lib()
    caps = [L.Lizard_compressBound(len(u)) for u in units] if caps is None else caps
    ptrs, sizes, held = _dict_args(dicts, len(units))
    return _batch(L.LizardB200_compress_dict_batch, units, caps, (level,), dicts=(ptrs, sizes))


def compress_using_dict(src: bytes, dict: bytes, level: int, cap: int = None, prefix: bool = False) -> bytes:
    """Lizard_createStream + Lizard_loadDict + Lizard_compress_continue on host bytes.  prefix=True lays the dictionary directly
    in front of the input; otherwise it is an external dictionary.  Returns b'' when the library returns 0."""
    L = lib()
    cap = L.Lizard_compressBound(len(src)) if cap is None else cap
    if prefix:
        buf = ctypes.create_string_buffer(bytes(dict) + bytes(src), len(dict) + len(src) + 1)
        dict_p, src_p = ctypes.addressof(buf), ctypes.addressof(buf) + len(dict)
    else:
        d = ctypes.create_string_buffer(bytes(dict), max(len(dict), 1))
        s = ctypes.create_string_buffer(bytes(src), max(len(src), 1))
        dict_p, src_p = ctypes.addressof(d), ctypes.addressof(s)
    dst = ctypes.create_string_buffer(max(cap, 1))
    st = L.Lizard_createStream(level)
    if not st:
        raise LizardB200Error("Lizard_createStream failed")
    try:
        L.Lizard_loadDict(st, dict_p, len(dict))
        n = L.Lizard_compress_continue(st, src_p, dst, len(src), cap)
    finally:
        L.Lizard_freeStream(st)
    return dst.raw[:n] if n > 0 else b""


def decompress_batch(units, caps):
    """LizardB200_decompress_batch: list of compressed bytes -> list of (result, bytes)."""
    return _batch(lib().LizardB200_decompress_batch, units, caps, ())


def decompress_partial_batch(units, targets, caps):
    """LizardB200_decompress_partial_batch: list of compressed bytes, per-unit targetOutputSize and capacity -> list of
    (result, bytes), each as decompress_partial."""
    if len(targets) != len(units):
        raise ValueError("one target per unit")
    return _batch(lib().LizardB200_decompress_partial_batch, units, caps, (), targets)


def decompress_dict_batch(units, dicts, caps):
    """LizardB200_decompress_dict_batch: list of compressed bytes, per-unit dictionary (bytes; b"" or None for none) and
    capacity -> list of (result, bytes), each as decompress_using_dict with an external dictionary.  Units given the same
    bytes object share one dictionary buffer."""
    ptrs, sizes, held = _dict_args(dicts, len(units))
    return _batch(lib().LizardB200_decompress_dict_batch, units, caps, (), dicts=(ptrs, sizes))


def _load_dg():
    global _dg
    if _dg is None:
        if not os.path.exists(DATAGEN_PATH):
            raise LizardB200Error(f"{DATAGEN_PATH} not built")
        _dg = ctypes.CDLL(DATAGEN_PATH)
        _dg.lizb200_datagen.argtypes = [ctypes.c_void_p, ctypes.c_ulonglong, ctypes.c_double, ctypes.c_double, ctypes.c_uint]
    return _dg


def datagen(size: int, match_pct: float = 50.0, seed: int = 0, lit_pct: float = 0.0) -> bytes:
    """Bytes identical to the reference's `datagen -g<size> -P<match_pct> -s<seed>` (tools/datagen.c)."""
    buf = ctypes.create_string_buffer(max(size, 1))
    if _load_dg().lizb200_datagen(buf, size, match_pct, lit_pct, seed) != 0:
        raise LizardB200Error("datagen failed")
    return buf.raw[:size]


def datagen_into(ptr: int, size: int, match_pct: float = 50.0, seed: int = 0, lit_pct: float = 0.0):
    """Same generator, writing into caller memory (e.g. a pinned torch tensor's data_ptr())."""
    if _load_dg().lizb200_datagen(ctypes.c_void_p(ptr), size, match_pct, lit_pct, seed) != 0:
        raise LizardB200Error("datagen failed")


# ---- frame layer (LizardF_*) -----------------------------------------------------------------------------------
class FrameInfo(ctypes.Structure):
    _fields_ = [("blockSizeID", ctypes.c_int), ("blockMode", ctypes.c_int), ("contentChecksumFlag", ctypes.c_int),
                ("frameType", ctypes.c_int), ("contentSize", ctypes.c_ulonglong), ("reserved", ctypes.c_uint * 2)]


class Preferences(ctypes.Structure):
    _fields_ = [("frameInfo", FrameInfo), ("compressionLevel", ctypes.c_int), ("autoFlush", ctypes.c_uint),
                ("reserved", ctypes.c_uint * 4)]


def make_prefs(level, block_id=1, independent=True, checksum=False, content_size=0):
    p = Preferences()
    p.frameInfo.blockSizeID = block_id
    p.frameInfo.blockMode = 1 if independent else 0
    p.frameInfo.contentChecksumFlag = 1 if checksum else 0
    p.frameInfo.contentSize = content_size
    p.compressionLevel = level
    return p


def bind_frame_api(L):
    """Set ctypes signatures of the LizardF_* symbols on a library handle (ours or the compiled reference)."""
    sz = ctypes.c_size_t
    L.LizardF_isError.argtypes = [sz]
    L.LizardF_getErrorName.argtypes = [sz]
    L.LizardF_getErrorName.restype = ctypes.c_char_p
    L.LizardF_compressFrameBound.restype = sz
    L.LizardF_compressFrameBound.argtypes = [sz, ctypes.c_void_p]
    L.LizardF_compressFrame.restype = sz
    L.LizardF_compressFrame.argtypes = [ctypes.c_void_p, sz, ctypes.c_void_p, sz, ctypes.c_void_p]
    L.LizardF_createCompressionContext.restype = sz
    L.LizardF_createCompressionContext.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    L.LizardF_freeCompressionContext.argtypes = [ctypes.c_void_p]
    for name in ("LizardF_compressBegin",):
        getattr(L, name).restype = sz
        getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p, sz, ctypes.c_void_p]
    L.LizardF_compressBound.restype = sz
    L.LizardF_compressBound.argtypes = [sz, ctypes.c_void_p]
    L.LizardF_compressUpdate.restype = sz
    L.LizardF_compressUpdate.argtypes = [ctypes.c_void_p, ctypes.c_void_p, sz, ctypes.c_void_p, sz, ctypes.c_void_p]
    for name in ("LizardF_flush", "LizardF_compressEnd"):
        getattr(L, name).restype = sz
        getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p, sz, ctypes.c_void_p]
    L.LizardF_createDecompressionContext.restype = sz
    L.LizardF_createDecompressionContext.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    L.LizardF_freeDecompressionContext.restype = sz
    L.LizardF_freeDecompressionContext.argtypes = [ctypes.c_void_p]
    L.LizardF_decompress.restype = sz
    L.LizardF_decompress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(sz), ctypes.c_void_p,
                                     ctypes.POINTER(sz), ctypes.c_void_p]
    L.LizardF_getFrameInfo.restype = sz
    L.LizardF_getFrameInfo.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(sz)]
    return L


def frame_compress(L, data: bytes, prefs) -> bytes:
    """LizardF_compressFrame on a library handle; raises on a frame error."""
    cap = L.LizardF_compressFrameBound(len(data), ctypes.byref(prefs))
    dst = ctypes.create_string_buffer(cap)
    n = L.LizardF_compressFrame(dst, cap, data, len(data), ctypes.byref(prefs))
    if L.LizardF_isError(n):
        raise LizardB200Error("LizardF_compressFrame: " + L.LizardF_getErrorName(n).decode())
    return dst.raw[:n]


def frame_decompress(L, frame: bytes, out_cap: int, chunk: int = 0, dst_chunk: int = 0):
    """Feed a frame to LizardF_decompress (whole, or in `chunk`-byte pieces). Returns (last result, bytes)."""
    ctx = ctypes.c_void_p()
    L.LizardF_createDecompressionContext(ctypes.byref(ctx), 100)
    out = ctypes.create_string_buffer(max(out_cap, 1))
    src = ctypes.create_string_buffer(frame, max(len(frame), 1))
    ip = op = 0
    res = 1
    try:
        while ip < len(frame) or res != 0:
            n_in = len(frame) - ip if not chunk else min(chunk, len(frame) - ip)
            n_out = out_cap - op if not dst_chunk else min(dst_chunk, out_cap - op)
            si = ctypes.c_size_t(n_in)
            so = ctypes.c_size_t(n_out)
            res = L.LizardF_decompress(ctx, ctypes.byref(out, op), ctypes.byref(so), ctypes.byref(src, ip),
                                       ctypes.byref(si), None)
            if L.LizardF_isError(res):
                return res, out.raw[:op]
            ip += si.value
            op += so.value
            if si.value == 0 and so.value == 0 and (n_in == 0 or n_out == 0):
                break
            if res == 0 and ip >= len(frame):
                break
    finally:
        L.LizardF_freeDecompressionContext(ctx)
    return res, out.raw[:op]


# ---- LizardF frames in device memory (LizardB200_compressFrames / LizardB200_decompressFrames) -----------------------
def _frame_tables(src_off, src_size, dst_off, dst_cap):
    n = len(src_off)
    if not (len(src_size) == len(dst_off) == len(dst_cap) == n):
        raise ValueError("one offset, size, destination offset and capacity per frame")
    u64 = ctypes.c_uint64 * n
    return n, u64(*src_off), u64(*src_size), u64(*dst_off), u64(*dst_cap), (ctypes.c_size_t * n)()


def compress_frames(d_src: int, src_off, src_size, d_dst: int, dst_off, dst_cap, prefs, stream: int = 0):
    """LizardB200_compressFrames: frame i is LizardF_compressFrame of the src_size[i] bytes at device address d_src + src_off[i],
    written to d_dst + dst_off[i] with room for dst_cap[i] bytes.  Addresses are integers (e.g. a tensor's data_ptr()), the
    tables host lists; `stream` is a cudaStream_t as an integer (0 = the default stream).  The call synchronises that stream.
    Returns the per-frame results (size_t: the frame size, or a LizardF error code, see frame_error)."""
    L = lib()
    n, so, ss, do, dc, res = _frame_tables(src_off, src_size, dst_off, dst_cap)
    _check(L.LizardB200_compressFrames(d_src, so, ss, d_dst, do, dc, res, n, ctypes.byref(prefs), stream or None),
           "LizardB200_compressFrames")
    return list(res)


def decompress_frames(d_src: int, src_off, src_size, d_dst: int, dst_off, dst_cap, stream: int = 0):
    """LizardB200_decompressFrames: frame i is the src_size[i] bytes at d_src + src_off[i], decoded to d_dst + dst_off[i] with
    room for dst_cap[i] bytes, as LizardF_decompress would in one call given all of it (include/lizard_b200.h).  Same argument
    conventions as compress_frames.  Returns the per-frame results (size_t: decoded size, 0 for a skippable frame, or a
    LizardF error code)."""
    L = lib()
    n, so, ss, do, dc, res = _frame_tables(src_off, src_size, dst_off, dst_cap)
    _check(L.LizardB200_decompressFrames(d_src, so, ss, d_dst, do, dc, res, n, stream or None), "LizardB200_decompressFrames")
    return list(res)


def _async_frame_args(args, n_frames, stream):
    """The device addresses, n_frames and stream of a device-table frame call: args are the source, its offset and size tables,
    the destination, its offset and capacity tables and the results, each a device address as an integer or a CUDA tensor."""
    ptr, stream = _device_args(args, stream)
    tables = [a for a in args[1:3] + args[4:] if not isinstance(a, int)]
    for a in tables:
        if a.element_size() != 8:
            raise ValueError("the offset, size and capacity tables and the results hold 8-byte integers")
    if n_frames is None:
        if not tables:
            raise ValueError("n_frames is needed when every table is an address")
        n_frames = tables[0].numel()
    for a in tables:
        if a.numel() < n_frames:
            raise ValueError("a table holds fewer entries than n_frames")
    return ptr, n_frames, stream


def _device_args(args, stream):
    """The device addresses of args (integers, or contiguous CUDA tensors) and the stream: None means the current torch stream
    of the first tensor, or 0 (the default stream) when every argument is an address."""
    tensors = [a for a in args if not isinstance(a, int)]
    for a in tensors:
        if not (a.is_cuda and a.is_contiguous()):
            raise ValueError("tensor arguments must be contiguous CUDA tensors")
    if stream is None:
        if tensors:
            import torch
            stream = torch.cuda.current_stream(tensors[0].device).cuda_stream
        else:
            stream = 0
    elif not isinstance(stream, int):
        stream = stream.cuda_stream
    return [a if isinstance(a, int) else a.data_ptr() for a in args], stream


def decompress_frames_async(d_src, d_src_off, d_src_size, d_dst, d_dst_off, d_dst_cap, d_result, max_blocks: int,
                            stage_bytes: int, stream=None, n_frames: int = None):
    """LizardB200_decompressFramesAsync: decompress_frames with the tables and the results in device memory, enqueue-only and
    capturable in a CUDA graph after one call of the same shape (include/lizard_b200.h).  Frames are admitted in index order
    while their blocks number at most max_blocks and their staging slots take at most stage_bytes; the others get
    ERROR_allocation_failed.  Every argument is a device address as an integer or a CUDA tensor (the tables 8-byte integers,
    one per frame; d_result 8 bytes per frame).  n_frames defaults to the length of a tensor table; `stream` to the current
    torch stream when tensors are given, else 0 (the default stream).  Returns nothing: read d_result after the stream's work."""
    ptr, n_frames, stream = _async_frame_args([d_src, d_src_off, d_src_size, d_dst, d_dst_off, d_dst_cap, d_result], n_frames,
                                              stream)
    _check(lib().LizardB200_decompressFramesAsync(*ptr, n_frames, max_blocks, stage_bytes, stream or None),
           "LizardB200_decompressFramesAsync")


def compress_frames_async(d_src, d_src_off, d_src_size, d_dst, d_dst_off, d_dst_cap, d_result, prefs, max_blocks: int,
                          stage_bytes: int, stream=None, n_frames: int = None):
    """LizardB200_compressFramesAsync: compress_frames with the tables and the results in device memory, enqueue-only and
    capturable in a CUDA graph after one call of the same shape (include/lizard_b200.h).  `prefs` is one Preferences for every
    frame (make_prefs; None = zeroed).  Frames are admitted in index order while their blocks number at most max_blocks and
    their staging bytes (each block's length rounded up to 16) take at most stage_bytes; the others get
    ERROR_allocation_failed.  Arguments, n_frames and `stream` as for decompress_frames_async.  Returns nothing: read d_result
    after the stream's work."""
    ptr, n_frames, stream = _async_frame_args([d_src, d_src_off, d_src_size, d_dst, d_dst_off, d_dst_cap, d_result], n_frames,
                                              stream)
    _check(lib().LizardB200_compressFramesAsync(*ptr, n_frames, ctypes.byref(prefs) if prefs is not None else None, max_blocks,
                                                stage_bytes, stream or None), "LizardB200_compressFramesAsync")


class DecompressionStream:
    """LizardB200_decompressStream: LizardF_decompress over device memory, one chunk per call, with its state kept between
    calls on the device current at creation (include/lizard_b200.h).  Use close() or a `with` block to free it."""

    def __init__(self):
        self._ds = ctypes.c_void_p()
        _check(lib().LizardB200_createDecompressionStream(ctypes.byref(self._ds)), "LizardB200_createDecompressionStream")

    def decompress(self, d_src, src_size: int, d_dst, dst_cap: int, stream=None):
        """Feed the src_size bytes at d_src with room for dst_cap bytes at d_dst (device addresses as integers, or contiguous
        CUDA tensors); `stream` as for decompress_frames_async (the current torch stream when tensors are given, else 0).  Returns (hint, consumed, produced): hint is LizardF_decompress's
        return value (a size_t; frame_error names an error)."""
        if self._ds is None:
            raise ValueError("the stream is closed")
        (src, dst), stream = _device_args([d_src, d_dst], stream)
        ss, ds = ctypes.c_size_t(src_size), ctypes.c_size_t(dst_cap)
        hint = lib().LizardB200_decompressStream(self._ds, dst, ctypes.byref(ds), src, ctypes.byref(ss), stream or None)
        return hint, ss.value, ds.value

    def close(self):
        if self._ds is not None:
            lib().LizardB200_freeDecompressionStream(self._ds)
            self._ds = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CompressionStream:
    """LizardB200_compressStream*: LizardF_compressBegin / Update / flush / End over device memory, with the stream's state kept
    between calls on the device current at creation (include/lizard_b200.h).  Addresses are integers or contiguous CUDA tensors;
    `stream` as for decompress_frames_async.  With d_written=None a method synchronises the stream and returns the call's result
    (a size or a LizardF error code, see frame_error); with a device address (8 bytes) it only enqueues and returns the host
    return value (0, or the error code of a refused call).  Use close() or a `with` block to free it."""

    def __init__(self):
        L = lib()
        self._cs = ctypes.c_void_p()
        _check(L.LizardB200_createCompressionStream(ctypes.byref(self._cs)), "LizardB200_createCompressionStream")

    def _call(self, fn, addrs, d_written, stream, args):
        """fn(stream object, *args(device addresses of addrs), dWritten, cudaStream)"""
        if self._cs is None:
            raise ValueError("the stream is closed")
        import torch
        own = None
        if d_written is None:
            t = next((a for a in addrs if not isinstance(a, int)), None)
            own = torch.empty(1, dtype=torch.int64, device=t.device if t is not None else "cuda")
        ptr, stream = _device_args(addrs + [d_written if own is None else own], stream)
        r = fn(self._cs, *args(ptr), ptr[-1], stream or None)
        if own is None or lib().LizardF_isError(r):
            return r
        if stream:
            torch.cuda.ExternalStream(stream).synchronize()
        else:
            torch.cuda.synchronize(own.device)
        return int(own.item()) & ((1 << 64) - 1)

    def begin(self, d_dst, dst_cap: int, prefs, d_written=None, stream=None):
        """LizardF_compressBegin: the frame header for `prefs` (a Preferences, make_prefs; None = zeroed) at d_dst."""
        p = ctypes.byref(prefs) if prefs is not None else None
        return self._call(lib().LizardB200_compressStreamBegin, [d_dst], d_written, stream, lambda a: (a[0], dst_cap, p))

    def update(self, d_src, src_size: int, d_dst, dst_cap: int, d_written=None, stream=None):
        """LizardF_compressUpdate: the src_size bytes at d_src, records to d_dst with room for dst_cap bytes."""
        return self._call(lib().LizardB200_compressStreamUpdate, [d_dst, d_src], d_written, stream,
                          lambda a: (a[0], dst_cap, a[1], src_size))

    def flush(self, d_dst, dst_cap: int, d_written=None, stream=None):
        """LizardF_flush: the carried partial block as a record."""
        return self._call(lib().LizardB200_compressStreamFlush, [d_dst], d_written, stream, lambda a: (a[0], dst_cap))

    def end(self, d_dst, dst_cap: int, d_written=None, stream=None):
        """LizardF_compressEnd: flush, the end mark and the content checksum."""
        return self._call(lib().LizardB200_compressStreamEnd, [d_dst], d_written, stream, lambda a: (a[0], dst_cap))

    def close(self):
        if self._cs is not None:
            lib().LizardB200_freeCompressionStream(self._cs)
            self._cs = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def frame_error(result: int):
    """None if a frame result is a size, else its LizardF error name (e.g. "ERROR_frameSize_wrong")."""
    L = lib()
    return L.LizardF_getErrorName(result).decode() if L.LizardF_isError(result) else None
