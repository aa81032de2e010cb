"""LizardB200_compressStream* (DESIGN.md 3.4e) on the CPU: the host build (lizard_b200/libhostshim.so, TEST-ONLY) of the shared
decisions (frame_cstream.h: frame_cbegin_run / frame_cupdate_run / frame_cflush_run / frame_cend_run) with the one-lane encoder in
place of the kernels, against the reference's LizardF_compressBegin / Update / flush / compressEnd call for call: every return
value and every byte written.

- Levels 10, 17, 21, 41 and 45; chunks of 0-19 bytes, random chunks, chunks of the block size - 1, exactly and + 1; autoFlush on
  and off; flushes mid-stream, one of them with a single carried byte; the content checksum on and off; contentSize right and
  wrong; a context reused after End.
- Every early return of the host calls, including the levels and the linked blocks this library refuses.
- The planning kernel's device function (cstream_unit) and the chunk split (frame_cupdate_plan) against a plain statement.
- The new kernels' registers, stack and local memory (cuobjdump -res-usage)."""
import ctypes
import os
import random
import re
import subprocess

import pytest

import lizard_b200 as lz
from tests import refs
from tests.test_encode_resources_cpu import _cuobjdump

SZ = ctypes.c_size_t
ULL = ctypes.c_ulonglong
LEVELS = (10, 17, 21, 41, 45)
BS = 128 << 10
ERR = {name: (1 << 64) - code for code, name in enumerate(
    ["OK", "GENERIC", "maxBlockSize_invalid", "blockMode_invalid", "contentChecksumFlag_invalid", "compressionLevel_invalid",
     "headerVersion_wrong", "blockChecksum_unsupported", "reservedFlag_set", "allocation_failed", "srcSize_tooLarge",
     "dstMaxSize_tooSmall"]) if code}


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
    vp = ctypes.c_void_p
    L.lzb_host_cstream_new.restype = vp
    L.lzb_host_cstream_free.argtypes = [vp]
    L.lzb_host_cstream_begin.argtypes = [vp, vp, SZ, vp]
    L.lzb_host_cstream_update.argtypes = [vp, vp, SZ, vp, SZ]
    L.lzb_host_cstream_flush.argtypes = [vp, vp, SZ]
    L.lzb_host_cstream_end.argtypes = [vp, vp, SZ]
    for f in ("begin", "update", "flush", "end"):
        getattr(L, "lzb_host_cstream_" + f).restype = SZ
    L.lzb_host_cstream_unit.argtypes = [ctypes.c_uint] + [ULL] * 6 + [ctypes.POINTER(ULL)]
    L.lzb_host_cupdate_plan.argtypes = [ULL, ULL, ctypes.c_uint, ULL, ctypes.POINTER(ULL)]
    return L


def is_err(r):
    return r > (1 << 64) - 20


class RefC:
    """The reference's LizardF_compress* on one context."""

    def __init__(self, L):
        self.L = L
        self.ctx = ctypes.c_void_p()
        L.LizardF_createCompressionContext(ctypes.byref(self.ctx), 100)

    def begin(self, dst, cap, prefs):
        return self.L.LizardF_compressBegin(self.ctx, dst, cap, ctypes.byref(prefs) if prefs is not None else None)

    def update(self, dst, cap, src, n):
        return self.L.LizardF_compressUpdate(self.ctx, dst, cap, src, n, None)

    def flush(self, dst, cap):
        return self.L.LizardF_flush(self.ctx, dst, cap, None)

    def end(self, dst, cap):
        return self.L.LizardF_compressEnd(self.ctx, dst, cap, None)

    def close(self):
        self.L.LizardF_freeCompressionContext(self.ctx)


class ShimC:
    """The shared decisions built in the host shim."""

    def __init__(self, S):
        self.S = S
        self.h = S.lzb_host_cstream_new()

    def begin(self, dst, cap, prefs):
        return self.S.lzb_host_cstream_begin(self.h, dst, cap, ctypes.byref(prefs) if prefs is not None else None)

    def update(self, dst, cap, src, n):
        return self.S.lzb_host_cstream_update(self.h, dst, cap, src, n)

    def flush(self, dst, cap):
        return self.S.lzb_host_cstream_flush(self.h, dst, cap)

    def end(self, dst, cap):
        return self.S.lzb_host_cstream_end(self.h, dst, cap)

    def close(self):
        self.S.lzb_host_cstream_free(self.h)


def bound(L, n, prefs):
    return L.LizardF_compressBound(n, ctypes.byref(prefs))


def run_calls(ctx, data, calls):
    """calls: ("begin", cap, prefs) / ("update", cap, offset, n) / ("flush", cap) / ("end", cap).  Returns [(result, bytes)]."""
    src = ctypes.create_string_buffer(data, max(len(data), 1))
    out = []
    for c in calls:
        cap = c[1]
        dst = ctypes.create_string_buffer(cap + 64)
        if c[0] == "begin":
            r = ctx.begin(dst, cap, c[2])
        elif c[0] == "update":
            r = ctx.update(dst, cap, ctypes.byref(src, c[2]), c[3])
        else:
            r = getattr(ctx, c[0])(dst, cap)
        out.append((r, b"" if is_err(r) else dst.raw[:r]))
    return out


def compare(ref, shim, data, calls):
    a, b = RefC(ref), ShimC(shim)
    try:
        ra, rb = run_calls(a, data, calls), run_calls(b, data, calls)
    finally:
        a.close()
        b.close()
    for k, (x, y) in enumerate(zip(ra, rb)):
        assert x == y, (k, calls[k][:1] + calls[k][2:] if calls[k][0] == "update" else calls[k], x[0], y[0])
    return ra


def chunked(ref, prefs, sizes, flush_at=()):
    """Begin, an Update per size, a flush after the updates listed in flush_at, End.  An Update's capacity is the bound, one byte
    more with autoFlush: a 1-byte last block's record is 10 bytes, one more than the bound counts without the checksum, and there
    the reference writes past its capacity where this library returns ERROR_dstMaxSize_tooSmall (test_one_byte_alone)."""
    calls = [("begin", 15, prefs)]
    off = 0
    for i, n in enumerate(sizes):
        calls.append(("update", bound(ref, n, prefs) + (1 if prefs.autoFlush else 0), off, n))
        off += n
        if i in flush_at:
            calls.append(("flush", BS + 8))
    calls.append(("end", BS + 16))
    return calls, off


@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("auto_flush", [0, 1])
@pytest.mark.parametrize("checksum", [False, True])
def test_chunk_patterns(ref, shim, level, auto_flush, checksum):
    data = lz.datagen(3 * BS + 5000, seed=level)
    rng = random.Random(level * 4 + auto_flush * 2 + checksum)
    patterns = [
        [n for n in range(20)] * 2,                                      # 0-19-byte chunks
        [BS - 1, BS, BS + 1],                                            # around the block size
        [rng.randrange(0, 70000) for _ in range(8)],                     # random chunks
    ]
    for sizes in patterns:
        p = lz.make_prefs(level, checksum=checksum)
        p.autoFlush = auto_flush
        calls, _ = chunked(ref, p, sizes, flush_at=(1, 3))
        res = compare(ref, shim, data, calls)
        assert not any(is_err(r) for r, _ in res)


@pytest.mark.parametrize("level", (10, 41))
def test_flush_of_one_carried_byte_and_content_size(ref, shim, level):
    data = lz.datagen(BS + 300, seed=7)
    for checksum in (False, True):
        for content_size in (BS + 21, BS + 22):                          # right, then wrong
            p = lz.make_prefs(level, checksum=checksum, content_size=content_size)
            # one carried byte: room for the carry + 7 is refused by both; its record is 10 bytes (test_one_byte_alone)
            calls = [("begin", 15, p), ("update", bound(ref, 1, p), 0, 1), ("flush", 1 + 7), ("flush", 10),
                     ("update", bound(ref, 1, p), 1, 1), ("flush", 10),
                     ("update", bound(ref, BS + 19, p), 2, BS + 19), ("end", 64)]
            res = compare(ref, shim, data, calls)
            assert is_err(res[-1][0]) == (content_size != BS + 21)


def test_reuse_after_end(ref, shim):
    data = lz.datagen(2 * BS, seed=3)
    p1, p2 = lz.make_prefs(21, checksum=True), lz.make_prefs(10, block_id=2)
    calls = []
    for p, sizes in ((p1, [5000, BS]), (p2, [BS + 7, 100]), (p1, [0, 1, 2])):
        c, _ = chunked(ref, p, sizes)
        calls += c
    compare(ref, shim, data, calls)


def test_early_returns(ref, shim):
    data = lz.datagen(BS + 64, seed=5)
    p = lz.make_prefs(17)
    b10 = bound(ref, 10, p)
    calls = [
        ("update", b10, 0, 10),                  # before Begin
        ("flush", 64), ("end", 64),              # nothing carried at stage 0: flush 0; End writes the end mark
        ("begin", 14, p),                        # dstMax < 15
        ("begin", 15, p), ("begin", 15, p),      # Begin twice
        ("update", b10 - 1, 0, 10),              # one byte below LizardF_compressBound
        ("update", b10, 0, 10),
        ("flush", 10 + 7),                       # room for the carry + 7
        ("flush", 10 + 8),
        ("flush", 64),                           # nothing carried
        ("end", 64), ("end", 64),
    ]
    res = compare(ref, shim, data, calls)
    assert res[0][0] == ERR["GENERIC"] and res[3][0] == ERR["dstMaxSize_tooSmall"] and res[5][0] == ERR["GENERIC"]
    assert res[6][0] == ERR["dstMaxSize_tooSmall"] and res[8][0] == ERR["dstMaxSize_tooSmall"]


def test_refused_preferences(shim):
    """Levels the encoder does not implement and linked blocks: this library refuses them at Begin (the reference does not)."""
    s = ShimC(shim)
    try:
        src = ctypes.create_string_buffer(b"x" * 100)
        cap = 1 << 18
        dst = ctypes.create_string_buffer(cap)
        for level in (12, 26, 49):
            assert s.begin(dst, 15, lz.make_prefs(level)) == ERR["compressionLevel_invalid"]
            assert s.update(dst, cap, src, 100) == ERR["GENERIC"]
        assert s.begin(dst, 15, lz.make_prefs(10, independent=False)) == ERR["blockMode_invalid"]
        bad = lz.make_prefs(10, block_id=0)
        bad.frameInfo.blockSizeID = 9
        assert s.begin(dst, 15, bad) == ERR["maxBlockSize_invalid"]
        assert s.begin(dst, 15, lz.make_prefs(10)) == 7
        assert s.update(dst, cap, src, 100) == 0
        assert s.end(dst, cap) > 100
    finally:
        s.close()


def test_one_byte_alone(ref, shim):
    """autoFlush and a 1-byte input: its record is 10 bytes, one more than the bound counts without the checksum.  This library
    refuses 9 bytes of room (the reference writes the tenth past it); from 10 bytes on both agree."""
    data = b"z" * 8
    for checksum in (False, True):
        p = lz.make_prefs(10, checksum=checksum)
        p.autoFlush = 1
        b1 = bound(ref, 1, p)
        if not checksum:
            s = ShimC(shim)
            try:
                dst = ctypes.create_string_buffer(64)
                assert s.begin(dst, 15, p) == 7 and s.update(dst, b1, data, 1) == ERR["dstMaxSize_tooSmall"]
                assert s.update(dst, b1 + 1, data, 1) == 10
            finally:
                s.close()
        compare(ref, shim, data, [("begin", 15, p), ("update", max(b1, 10), 0, 1), ("update", b1 + 1, 1, 1), ("end", 16)])


def test_block_split(shim):
    """cstream_unit against a plain statement: the carried block first, then the chunk's blocks, the last one shorter."""
    out = (ULL * 4)()
    stride = 1 << 20
    for bs in (BS, 4 << 20):
        for carry_len in (0, 1, bs - 1, bs):
            for n in (0, 1, bs - 1, bs, bs + 1, 3 * bs - 1, 3 * bs, 3 * bs + 1):
                units = (1 if carry_len else 0) + -(-n // bs)
                want = []
                if carry_len:
                    want.append((7777, carry_len))
                want += [(10 ** 9 + i, min(bs, n - i)) for i in range(0, n, bs)]
                assert len(want) == units
                for k, (s, ln) in enumerate(want):
                    shim.lzb_host_cstream_unit(k, 7777, carry_len, 10 ** 9, n, bs, stride, out)
                    assert tuple(out) == (s, ln, k * stride, ln - 1), (bs, carry_len, n, k)


def test_chunk_split(shim):
    """frame_cupdate_plan: what completes the carried block, the whole blocks (autoFlush: all the rest), the remainder."""
    out = (ULL * 4)()
    for bs in (BS, 1 << 20):
        for carry in (0, 1, bs - 1):
            for n in (0, 1, bs - carry - 1, bs - carry, bs - carry + 1, 2 * bs, 5 * bs + 3):
                for af in (0, 1):
                    shim.lzb_host_cupdate_plan(carry, bs, af, n, out)
                    take = min(n, bs - carry) if carry else 0
                    left = n - take
                    whole = left if af else left // bs * bs
                    assert tuple(out) == (take, whole, left - whole, 1 if carry and take == bs - carry else 0)


# registers, stack bytes; local memory must be 0
CSTREAM_KERNEL_LIMITS = {
    "lizard_cstream_begin_kernel": (40, 0),
    "lizard_cstream_plan_kernel": (32, 0),
    "lizard_cstream_scan_kernel": (40, 0),
    "lizard_cstream_assemble_kernel": (48, 0),
    "lizard_cstream_hash_kernel": (48, 0),
    "lizard_cstream_finish_kernel": (40, 0),
}


def test_cstream_kernel_resources():
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
            for k in CSTREAM_KERNEL_LIMITS:
                if re.search(r"\d" + k + r"[A-Z]", name):
                    found[k] = {a: int(b) for a, b in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    assert set(found) == set(CSTREAM_KERNEL_LIMITS), found
    for k, (reg, stack) in CSTREAM_KERNEL_LIMITS.items():
        r = found[k]
        assert r["REG"] <= reg and r["STACK"] <= stack and r["LOCAL"] == 0, (k, r)
