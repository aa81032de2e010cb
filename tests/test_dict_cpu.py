"""Lizard_decompress_safe_usingDict through the device decoder's code on the CPU: the one-lane host build and the 32-lane warp
emulator of the dictionary kernel (lizard_b200/libhostshim.so, TEST-ONLY) against the compiled reference.  The streams come
from the reference's own dictionary compressor (Lizard_loadDict + Lizard_compress_continue), in the two layouts its decoder
tells apart (lib/lizard_decompress.c:351-360): the dictionary directly in front of the output (read in place), and a
dictionary somewhere else (an external dictionary).  Return codes must be equal, decoded bytes must be the input, and
nothing may be written outside [dst, dst + cap) or into the dictionary.

The shim takes what the kernel takes: the dictionary's end, the bytes readable in front of it, and the reach of the
reference's offset check (dict_reach below).  Also checked here: every decode kernel instance that existed before the
dictionary kernel compiles to the same SASS, and the dictionary kernel's resources are pinned."""
import ctypes
import functools
import hashlib
import os
import random
import re
import subprocess

import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_encode_resources_cpu import _cuobjdump

BS = lz.BLOCK_SIZE
HOST, EMU = "lzb_host_decompress_dict", "lzb_emu_decompress_dict"
GUARD = 64
UNCHECKED = 0xFFFFFFFF
PREFIX_MAX = (1 << 24) - 1


def dict_reach(size, prefix):
    """How far below the unit start a match may start before the reference's offset check fails (decode.cuh dict_reach)."""
    if prefix:
        return 1 << 24 if size >= PREFIX_MAX else size
    return UNCHECKED if size >= 1 << 24 else size


def dict_window(level):
    return PREFIX_MAX if corpus.is_lizv1(level) else 65535


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    vp, ci = ctypes.c_void_p, ctypes.c_int
    L.Lizard_createStream.restype = vp
    L.Lizard_createStream.argtypes = [ci]
    L.Lizard_freeStream.argtypes = [vp]
    L.Lizard_loadDict.argtypes = [vp, vp, ci]
    L.Lizard_compress_continue.argtypes = [vp, vp, vp, ci, ci]
    L.Lizard_decompress_safe_usingDict.argtypes = [vp, vp, ci, ci, vp, ci]
    L.Lizard_createStreamDecode.restype = vp
    L.Lizard_freeStreamDecode.argtypes = [vp]
    L.Lizard_setStreamDecode.argtypes = [vp, vp, ci]
    L.Lizard_decompress_safe_continue.argtypes = [vp, vp, vp, ci, ci]
    return L


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    for f in (HOST, EMU):
        getattr(L, f).argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint,
                                  ctypes.c_uint]
    L.lzb_dict_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)] * 2 + [ctypes.c_int]
    L.lzb_emu_lane_order.argtypes = [ctypes.c_int]
    return L


def stats(shim, reset=True):
    a, b = ctypes.c_ulonglong(), ctypes.c_ulonglong()
    shim.lzb_dict_stats(ctypes.byref(a), ctypes.byref(b), 1 if reset else 0)
    return a.value, b.value


# ---- the reference's side ------------------------------------------------------------------------------------------
def ref_compress_dict(ref, dictionary, data, level, prefix):
    """Lizard_loadDict + Lizard_compress_continue: in place (dictionary and input in one buffer) or with the input elsewhere."""
    st = ref.Lizard_createStream(level)
    cap = len(data) + len(data) // 8 + 1024
    out = ctypes.create_string_buffer(cap)
    if prefix:
        buf = ctypes.create_string_buffer(dictionary + data, len(dictionary) + len(data) + 1)
        ref.Lizard_loadDict(st, buf, len(dictionary))
        n = ref.Lizard_compress_continue(st, ctypes.addressof(buf) + len(dictionary), out, len(data), cap)
    else:
        dbuf = ctypes.create_string_buffer(dictionary, len(dictionary) + 1)
        sbuf = ctypes.create_string_buffer(data, len(data) + 1)
        ref.Lizard_loadDict(st, dbuf, len(dictionary))
        n = ref.Lizard_compress_continue(st, sbuf, out, len(data), cap)
    ref.Lizard_freeStream(st)
    assert n > 0, (level, prefix, len(data))
    return out.raw[:n]


def ref_decode_dict(ref, comp, dictionary, cap, prefix):
    room = 2 * max(cap, 1) + 64                               # the reference's wild copies and raw-block overrun (DESIGN 3.5)
    if prefix:
        buf = ctypes.create_string_buffer(dictionary, len(dictionary) + room)
        dst = ctypes.addressof(buf) + len(dictionary)
        r = ref.Lizard_decompress_safe_usingDict(comp, dst, len(comp), cap, ctypes.addressof(buf), len(dictionary))
    else:
        dbuf = ctypes.create_string_buffer(dictionary, max(len(dictionary), 1))
        buf = ctypes.create_string_buffer(room)
        dst = ctypes.addressof(buf)
        r = ref.Lizard_decompress_safe_usingDict(comp, dst, len(comp), cap, dbuf, len(dictionary))
    return r, ctypes.string_at(dst, max(r, 0))


# ---- the device code's side ----------------------------------------------------------------------------------------
def dev_decode_dict(shim, fn, comp, dictionary, cap, prefix, reach=None, avail=None):
    """One call of the shim with guard bytes behind the capacity; the dictionary must come back unchanged."""
    level = comp[0] if comp else 10
    size = len(dictionary)
    reach = dict_reach(size, prefix) if reach is None else reach
    avail = min(size, dict_window(level)) if avail is None else avail
    if prefix:
        buf = ctypes.create_string_buffer(dictionary + b"\xA5" * (cap + GUARD), size + cap + GUARD)
        base, dst = ctypes.addressof(buf), ctypes.addressof(buf) + size
        end = dst
    else:
        dbuf = ctypes.create_string_buffer(dictionary, max(size, 1))
        buf = ctypes.create_string_buffer(b"\xA5" * (cap + GUARD), cap + GUARD)
        base, dst = ctypes.addressof(dbuf), ctypes.addressof(buf)
        end = base + size
    r = getattr(shim, fn)(comp, len(comp), dst, cap, end, avail, reach)
    assert ctypes.string_at(dst + cap, GUARD) == b"\xA5" * GUARD, (fn, cap, "wrote behind the capacity")
    assert ctypes.string_at(base, size) == dictionary, (fn, "wrote into the dictionary")
    return r, ctypes.string_at(dst, max(r, 0))


def check(ref, shim, comp, dictionary, cap, prefix, data=None, fns=(HOST, EMU), orders=(0,)):
    rr, ro = ref_decode_dict(ref, comp, dictionary, cap, prefix)
    for fn in fns:
        for o in (orders if fn == EMU else (0,)):
            shim.lzb_emu_lane_order(o)
            r, out = dev_decode_dict(shim, fn, comp, dictionary, cap, prefix)
            assert r == rr, (fn, o, prefix, len(comp), len(dictionary), cap, r, rr)
            if data is not None and rr > 0:
                assert out == ro == data, (fn, o, prefix, len(comp), len(dictionary))
    shim.lzb_emu_lane_order(0)
    return rr


# ---- inputs ----------------------------------------------------------------------------------------------------------
def records(n_bytes, seed):
    """JSON-like records drawn from a fixed vocabulary: what shared dictionaries are for."""
    rnd = random.Random(seed)
    keys = ["id", "name", "email", "status", "created_at", "tags", "score", "country", "device", "session"]
    words = ["alpha", "bravo", "charlie", "delta", "echo", "foxtrot", "golf", "hotel", "india", "juliet", "active",
             "pending", "closed", "mobile", "desktop", "DE", "FR", "US", "JP", "premium", "basic"]
    out = bytearray()
    while len(out) < n_bytes:
        fields = rnd.sample(keys, rnd.randint(4, len(keys)))
        parts = []
        for k in fields:
            v = rnd.choice([str(rnd.randrange(10 ** rnd.randint(1, 8))), '"%s"' % rnd.choice(words),
                            '["%s","%s"]' % (rnd.choice(words), rnd.choice(words))])
            parts.append('"%s":%s' % (k, v))
        out += ("{" + ",".join(parts) + "}\n").encode()
    return bytes(out[:n_bytes])


@functools.lru_cache(maxsize=None)
def _dictionary(size=1 << 16):
    return records(size, 12345)


def _straddler(dictionary, seed):
    """A unit that starts with a piece it repeats right behind the dictionary's last bytes: the compressor finds one match
    that starts in the dictionary and runs into the unit."""
    a = records(300, seed)
    return a + dictionary[-40:] + a + records(200, seed + 1)


@functools.lru_cache(maxsize=None)
def _level_inputs(level):
    d = _dictionary()
    return [_straddler(d, level), records(6000, 100 + level), d[5000:9000] + records(3000, 200 + level) + d[-2000:]]


# ---- tests -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", range(10, 50))
def test_every_level_matches_reference(ref, shim, level):
    """Every level 10-49, both layouts: the one-lane build and the emulator (forward, reverse and shuffled lane orders) return
    what the reference returns and decode the input; a capacity one byte short fails where the reference fails."""
    d = _dictionary()
    for prefix in (True, False):
        for data in _level_inputs(level):
            comp = ref_compress_dict(ref, d, data, level, prefix)
            check(ref, shim, comp, d, len(data), prefix, data, orders=(0, 1, 2))
            check(ref, shim, comp, d, len(data) - 1, prefix, fns=(HOST,))


# The reference's fast parsers (levels 10, 11, 30, 31) do not search a loaded dictionary; every other parser does.
@pytest.mark.parametrize("flavour,levels", [("fastLZ4", (13, 17, 19, 35, 38)), ("LIZv1", (20, 21, 26, 41, 45))])
def test_every_codeword_flavour_reads_and_straddles_the_dictionary(ref, shim, flavour, levels):
    """Not vacuous: in both layouts, the one-lane build and the emulator decode matches that lie wholly in the dictionary and
    matches that start in it and run into the unit (the shim counts both kinds)."""
    d = _dictionary()
    for prefix in (True, False):
        for fn in (HOST, EMU):
            stats(shim)
            for level in levels:
                for data in _level_inputs(level):
                    check(ref, shim, ref_compress_dict(ref, d, data, level, prefix), d, len(data), prefix, data, fns=(fn,))
            only, straddle = stats(shim)
            assert only > 0 and straddle > 0, (flavour, prefix, fn, only, straddle)


@pytest.mark.parametrize("level", [10, 21, 41])
def test_units_of_several_inner_blocks(ref, shim, level):
    """A unit of two inner blocks: the dictionary stays reachable from the second block (lowLimit is fixed per call)."""
    d = _dictionary()
    data = records(BS + 9000, 77) + d[100:3000]
    for prefix in (True, False):
        comp = ref_compress_dict(ref, d, data, level, prefix)
        check(ref, shim, comp, d, len(data), prefix, data, fns=(HOST,))


def _shortest_dictionary(ref, comp, d, cap, prefix):
    """The fewest trailing dictionary bytes with which the reference still decodes the unit."""
    lo, hi = 0, len(d)
    while lo < hi:
        mid = (lo + hi) // 2
        if ref_decode_dict(ref, comp, d[len(d) - mid:], cap, prefix)[0] > 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("level", [13, 17, 20, 21, 35, 41, 45])
def test_reach_edges(ref, shim, level):
    """The dictionary shortened from its front: with exactly the bytes the farthest match needs the unit decodes, one byte
    fewer gives the reference's token error (-(token index)-1) at the first match that reaches too far."""
    d = _dictionary()
    data = _level_inputs(level)[2]
    for prefix in (True, False):
        comp = ref_compress_dict(ref, d, data, level, prefix)
        need = _shortest_dictionary(ref, comp, d, len(data), prefix)
        assert 0 < need <= len(d), need
        for k in (need, need - 1, need // 2, 1):
            r = check(ref, shim, comp, d[len(d) - k:], len(data), prefix, data if k >= need else None, orders=(0, 2))
            if k < need:
                assert r < -1, (k, need, r)                     # a token error, not the header / stream error -1


def _long_offset_unit(level, off, ml_code=5, lead=0):
    """A LIZv1 unit of one inner block, all streams raw: one 24-bit-offset token (match length ml_code + 16) at the unit start,
    then 16 literals.  Its match starts `off` bytes below the unit start.  lead = 1..7: in front of it a token of `lead`
    literals and an 8-byte match at 16-bit offset 1000, so the far match starts off - lead - 8 bytes below the unit start."""
    le24 = lambda v: bytes([v & 255, (v >> 8) & 255, v >> 16])
    lits = bytes(range(65 - lead, 81))
    off16 = bytes([1000 & 255, 1000 >> 8]) if lead else b""
    flags = (bytes([(8 << 3) | lead]) if lead else b"") + bytes([ml_code])
    body = (le24(0) + le24(len(off16)) + off16 + le24(3) + le24(off) + le24(len(flags)) + flags + le24(len(lits)) + lits)
    return bytes([level, 0]) + body, (lead + 8 if lead else 0) + ml_code + 16 + 16


@pytest.mark.parametrize("prefix", [True, False])
def test_the_2_24_switches(ref, shim, prefix):
    """An offset of 2^24 - 1 at the unit start.  In place, a dictionary of 2^24 - 2 bytes checks it against its size (token
    error), one of 2^24 - 1 bytes switches to the reference's withPrefix64k (lowPrefix = dest - 2^24) and passes.  External,
    2^24 - 1 bytes pass the check exactly and 2^24 bytes or more switch the check off."""
    big = bytes(random.Random(7).getrandbits(8) for _ in range(1 << 12)) * ((1 << 24) // (1 << 12) + 1)
    comp, n = _long_offset_unit(20, PREFIX_MAX)
    for size in ((1 << 24) - 2, PREFIX_MAX, 1 << 24, (1 << 24) + 5):
        d = big[:size]
        rr, ro = ref_decode_dict(ref, comp, d, n + 16, prefix)
        assert rr == (-2 if size < PREFIX_MAX else n), (size, rr)
        for fn in (HOST, EMU):
            r, out = dev_decode_dict(shim, fn, comp, d, n + 16, prefix)
            assert (r, out) == (rr, ro), (fn, size, r, rr)
        if rr > 0:
            assert ro[:21] == d[-PREFIX_MAX:][:21]
    # dictionaries at the LZ4 codewords' 16-bit window: only the last 65535 bytes are ever read
    d = _dictionary(1 << 17)
    data = _level_inputs(10)[2]
    comp = ref_compress_dict(ref, d, data, 10, prefix)
    assert dev_decode_dict(shim, HOST, comp, d, len(data), prefix, avail=65535)[1] == data


def _linked_stream(ref, data, level, piece, double_buffer, place=None, load=None):
    """The reference's streamed compression: Lizard_compress_continue on consecutive pieces of one buffer, or on pieces
    copied into two buffers in turn (each piece then sees only the one before it, lizard_compress.c:439-449), or on pieces
    copied to the addresses place(k) that the caller chooses (so the compressor sees the layout a decoder will use).
    load = (address, size): Lizard_loadDict of those bytes first."""
    st = ref.Lizard_createStream(level)
    if load:
        ref.Lizard_loadDict(st, load[0], load[1])
    src = ctypes.create_string_buffer(data, len(data) + 1)
    two = [ctypes.create_string_buffer(piece + 1) for _ in range(2)]
    out = []
    for at in range(0, len(data), piece):
        n_in = min(piece, len(data) - at)
        cap = n_in + n_in // 8 + 1024
        buf = ctypes.create_string_buffer(cap)
        where = ctypes.addressof(src) + at
        if double_buffer or place:
            where = place(at // piece) if place else ctypes.addressof(two[(at // piece) % 2])
            ctypes.memmove(where, data[at:at + n_in], n_in)
        n = ref.Lizard_compress_continue(st, where, buf, n_in, cap)
        assert n > 0
        out.append((buf.raw[:n], n_in))
    ref.Lizard_freeStream(st)
    return out


class _Window:
    """Lizard_decompress_safe_continue's state (lib/lizard_decompress.c:303-344), decoding through the shim as the library
    does: the reachable tail of [external dictionary][prefix] gathered into one buffer, reach = the whole window."""

    def __init__(self):
        self.ext, self.ext_size, self.pre_end, self.pre_size = 0, 0, 0, 0

    def set(self, addr, size):
        self.pre_size, self.pre_end, self.ext, self.ext_size = size, addr + size, 0, 0

    def decode(self, shim, fn, comp, dst, cap):
        if self.pre_end == dst:
            ext, ext_size, pre, pre_size = self.ext, self.ext_size, self.pre_end - self.pre_size, self.pre_size
        else:
            self.ext_size, self.ext = self.pre_size, self.pre_end - self.pre_size
            ext, ext_size, pre, pre_size = self.ext, self.ext_size, 0, 0
        total = ext_size + pre_size
        keep = min(total, dict_window(comp[0]))
        from_pre = min(keep, pre_size)
        win = ctypes.string_at(ext + ext_size - (keep - from_pre), keep - from_pre) + ctypes.string_at(pre + pre_size - from_pre, from_pre)
        wbuf = ctypes.create_string_buffer(win, max(len(win), 1))
        reach = UNCHECKED if total >= 1 << 24 else total
        r = getattr(shim, fn)(comp, len(comp), dst, cap, ctypes.addressof(wbuf) + len(win), len(win), reach)
        if r > 0:
            if self.pre_end == dst:
                self.pre_size += r
                self.pre_end += r
            else:
                self.pre_size, self.pre_end = r, dst + r
        return r


@pytest.mark.parametrize("level", [10, 21, 41])
@pytest.mark.parametrize("layout", ["contiguous", "double_buffer", "saved_copy"])
def test_continue_sequences(ref, shim, level, layout):
    """A linked stream of 8 KiB pieces, decoded piece by piece the three ways the reference's _continue supports: into one
    contiguous buffer (the prefix grows in place), alternating between two buffers (every call takes the external-dictionary
    branch), and after Lizard_setStreamDecode to a saved copy of the last 16 KiB.  The last two decode a stream that was
    compressed from two alternating buffers, whose matches reach one piece back.  The reference and the shim walk the same
    sequence; every return code must agree and the output must be the input."""
    data = records(96 << 10, 900 + level)
    pieces = _linked_stream(ref, data, level, 8 << 10, layout != "contiguous")
    for who in ("ref", HOST):
        total = ctypes.create_string_buffer(len(data) + 64)
        bufs = [ctypes.create_string_buffer((8 << 10) + 64) for _ in range(2)]
        saved = ctypes.create_string_buffer(16 << 10)
        sd = ref.Lizard_createStreamDecode() if who == "ref" else None
        win = _Window()
        if who == "ref":
            ref.Lizard_setStreamDecode(sd, None, 0)
        out, at = b"", 0
        for k, (comp, n_in) in enumerate(pieces):
            if layout == "contiguous":
                dst = ctypes.addressof(total) + at
            else:
                dst = ctypes.addressof(bufs[k % 2])
            if layout == "saved_copy" and k > 0:
                keep = min(len(out), 16 << 10)
                ctypes.memmove(saved, out[len(out) - keep:], keep)
                if who == "ref":
                    ref.Lizard_setStreamDecode(sd, saved, keep)
                else:
                    win.set(ctypes.addressof(saved), keep)
                dst = ctypes.addressof(bufs[k % 2])
            if who == "ref":
                r = ref.Lizard_decompress_safe_continue(sd, comp, dst, len(comp), n_in)
            else:
                r = win.decode(shim, HOST, comp, dst, n_in)
            assert r == n_in, (who, layout, k, r)
            out += ctypes.string_at(dst, r)
            at += r
        if sd:
            ref.Lizard_freeStreamDecode(sd)
        assert out == data, (who, layout)


def _damage(rnd, comp):
    b = bytearray(comp)
    for _ in range(rnd.choice([1, 1, 2])):
        at = rnd.randrange(1, len(b))
        b[at] ^= (1 << rnd.randrange(8)) if rnd.random() < 0.5 else rnd.randrange(1, 256)
    return bytes(b)


@pytest.mark.parametrize("level", [10, 20, 21, 30, 41])
def test_damaged_streams(ref, shim, level):
    """Truncations and bit flips, in front of and behind the dictionary matches (the straddler's dictionary match is its
    first): return codes equal to the reference's.  Bytes are not compared, because damage can create offsets below 8,
    where the reference's output depends on stale memory (DESIGN.md 3.5)."""
    rnd = random.Random(500 + level)
    d = _dictionary()
    failed = 0
    for prefix in (True, False):
        for data in _level_inputs(level)[:2]:
            comp = ref_compress_dict(ref, d, data, level, prefix)
            for cut in (1, 2, len(comp) // 3, len(comp) - 1):
                failed += check(ref, shim, comp[:cut], d, len(data), prefix, fns=(HOST,)) < 0
            for _ in range(12):
                failed += check(ref, shim, _damage(rnd, comp), d, len(data), prefix, fns=(HOST, EMU)) < 0
    assert failed > 10, failed


def test_no_dictionary_is_decompress_safe(ref, shim):
    """Reach 0 and no readable bytes: the dictionary kernel decodes plain units as Lizard_decompress_safe, offsets reaching
    below the unit start included."""
    for level in (17, 21, 41):                                # parsers that search a loaded dictionary
        data = records(20000, level)
        comp = refs.ref_compress(ref, data, level)
        for fn in (HOST, EMU):
            assert dev_decode_dict(shim, fn, comp, b"", len(data), False) == (len(data), data)
        d = _dictionary()
        comp = ref_compress_dict(ref, d, _straddler(d, level), level, False)
        want = refs.ref_decompress(ref, comp, 4000)[0]
        assert want < -1
        assert dev_decode_dict(shim, HOST, comp, b"", 4000, False)[0] == want


# ---------------------------------------------------------------------------------------------------------------------
# compiled kernels
# ---------------------------------------------------------------------------------------------------------------------
# SHA-256 of the instructions (cuobjdump -sass, addresses and encodings included) of every decode kernel instance that
# existed before the dictionary kernel: adding it must not change their code.  (sm_90a, CUDA 12.9)
SASS_BEFORE_DICT = {
    "lizard_decode_units_kernelILi0EE": "d03bbda13a6e7920",
    "lizard_decode_units_kernelILi1EE": "5a00a6832b7cdc3e",
    "lizard_decode_units_kernelILi2EE": "1f030309e6afd373",
    "lizard_decode_units_kernelILi3EE": "dbe49ad557b6d933",
    "lizard_decode_partial_units_kernel": "a6b35edaad5dd907",
    "lizard_decode2_units_kernelILj4EE": "9f1cb3e60e15298e",
    "lizard_decode2_units_kernelILj8EE": "3b29b2f178daa6e5",
    "lizard_huf_plan_kernel": "af80fdcd8c0b96fd",
    "lizard_huf_expand_kernel": "8ad99dba0af6f8fe",
    "lizard_token_parse_kernel": "c61c9b72eeeb6492",
    "lizard_gather_segments_kernel": "ce19d7b07c201586",
    "lizard_encode_units_kernelILi0EE": "50112e71fcdbc5ec",
    "lizard_encode_units_kernelILi1EE": "0ea0914d23166bfa",
    "lizard_encode_units_kernelILi2EE": "d5c06ae07eba5543",
}


def _sass_by_kernel():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    lib = os.path.join(refs.ROOT, "lizard_b200", "liblizard_b200.so")
    out = subprocess.run([exe, "-sass", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    return sass_digests(out)


def sass_digests(text):
    """kernel name and template arguments (not the anonymous-namespace tag, which follows the source file) -> digest of its
    instruction lines"""
    found, name, lines = {}, None, []
    for line in text.splitlines() + ["Function : lizard_end_kernel"]:
        m = re.search(r"Function : \S*?(lizard_\w+?_kernel(?:IL[ij]\d+EE)?)", line)
        if m:
            if name:
                found[name] = hashlib.sha256("\n".join(lines).encode()).hexdigest()[:16]
            name = m.group(1)
            lines = []
        elif name and re.search(r"/\*[0-9a-f]{4}\*/", line):
            lines.append(line.strip())
    return found


def test_existing_decode_kernels_compile_to_the_same_sass():
    got = _sass_by_kernel()
    assert SASS_BEFORE_DICT, "no pinned digests"
    for k, want in SASS_BEFORE_DICT.items():
        assert got.get(k) == want, (k, got.get(k), want)


def test_dictionary_kernel_is_its_own_instance_within_the_token_kernels_registers():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    lib = os.path.join(refs.ROOT, "lizard_b200", "liblizard_b200.so")
    out = subprocess.run([exe, "-res-usage", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    res, name = None, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "lizard_decode_dict_units_kernel" in name and "REG:" in line:
            res = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    assert res is not None, "lizard_decode_dict_units_kernel not in the library"
    assert res == DICT_KERNEL, res


DICT_KERNEL = {"REG": 64, "STACK": 688, "SHARED": 1024, "LOCAL": 0}       # (sm_90a, CUDA 12.9)


def test_binding_signatures_match_the_header():
    """The ctypes signatures of the dictionary calls have as many arguments as their prototypes in include/lizard_b200.h
    (a pointer bound as an integer would be truncated)."""
    header = open(os.path.join(refs.ROOT, "include", "lizard_b200.h")).read()
    L = lz.lib()
    for name in ("LizardB200_decompress_dict_device", "LizardB200_decompress_dict_batch", "Lizard_decompress_safe_usingDict",
                 "Lizard_setStreamDecode", "Lizard_decompress_safe_continue"):
        m = re.search(r"\b%s\s*\(([^)]*)\)\s*;" % name, header)
        assert m, name
        params = [p for p in m.group(1).split(",") if p.strip()]
        assert len(getattr(L, name).argtypes) == len(params), (name, len(params))
        pointers = [("*" in p) for p in params]
        kinds = [t in (ctypes.c_void_p, ctypes.c_char_p) or hasattr(t, "contents") or t.__name__.startswith("LP_")
                 for t in getattr(L, name).argtypes]
        assert kinds == pointers, (name, kinds, pointers)
