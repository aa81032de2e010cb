"""LizardB200_compressFramesAsync (DESIGN.md 3.4c) on the CPU: the host build (lizard_b200/libhostshim.so, TEST-ONLY) of the
per-frame decisions its planning kernels run, and of its admission.

- frame_compress_plan (frame_device.cuh) gives what this library's LizardF_compressFrameBound and LizardF_compressBegin give on
  LizardF_compressFrame's preferences, and the reference's LizardF_compressFrame header bytes: every block size ID 0-8, both
  block modes, with and without the content checksum and the content size, a level the GPU runs and a refused one; sizes 0, 1,
  2, every block size -1 / +0 / +1 and beyond 4 GiB; capacities at the bound -1 / +0 / +1.
- The planning admits the prefix a plain statement of the rule gives: bounds that end exactly at frame k's blocks or staging
  bytes and one below, frames that take nothing in front of and behind the cut, and the stage clamp up to SIZE_MAX.
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

U64 = ctypes.c_ulonglong
KB, MB, GB = 1 << 10, 1 << 20, 1 << 30
BLOCK = {1: 128 * KB, 2: 256 * KB, 3: 1 * MB, 4: 4 * MB, 5: 16 * MB, 6: 64 * MB, 7: 256 * MB}
ERR_BLOCK_SIZE = (1 << 64) - 2                    # frame_block_size of an invalid ID: LizardF_ERROR_maxBlockSize_invalid
TOO_SMALL = 11
GPU_LEVEL, REFUSED_LEVEL = 10, 12
SIZE_MAX = (1 << 64) - 1


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    L.lzb_host_frame_compress_plan.argtypes = [ctypes.c_uint] * 4 + [U64, ctypes.c_int, U64, U64, ctypes.c_void_p,
                                                                      ctypes.c_void_p]
    L.lzb_host_frame_compress_plan.restype = ctypes.c_uint
    L.lzb_host_frame_compress_stage_limit.argtypes = [ctypes.c_uint, ctypes.c_uint, U64]
    L.lzb_host_frame_compress_stage_limit.restype = U64
    L.lzb_host_frame_compress_admit.argtypes = [ctypes.c_uint, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint, ctypes.c_uint,
                                                ctypes.c_uint, U64, ctypes.c_int, ctypes.c_uint, U64, ctypes.c_void_p,
                                                ctypes.c_void_p, ctypes.c_void_p]
    return L


@pytest.fixture(scope="module")
def ours():
    try:
        return lz.bind_frame_api(lz.lib())
    except lz.LizardB200Error:
        pytest.skip("liblizard_b200.so not built")


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return lz.bind_frame_api(L)


def block_size(bsid):
    return BLOCK.get(1 if bsid == 0 else bsid, ERR_BLOCK_SIZE)


def one_shot(bsid, mode, checksum, csize, n):
    """LizardF_compressFrame's preferences for an n-byte frame, stated plainly (lizard_frame.c:260-290)."""
    prop = 1
    while bsid > prop:
        if n <= block_size(prop):
            bsid = prop
            break
        prop += 1
    p = lz.make_prefs(GPU_LEVEL, bsid, mode == 1 or n <= block_size(bsid), checksum, n if csize else 0)
    p.autoFlush = 1
    return p


def plan(shim, bsid, mode, checksum, csize, level_ok, n, cap):
    hdr = ctypes.create_string_buffer(16)
    out = (U64 * 5)()
    v = shim.lzb_host_frame_compress_plan(bsid, mode, int(checksum), 0, csize, int(level_ok), n, cap, hdr, out)
    return v, hdr.raw[:out[0]], list(out)


def sizes_to_check():
    s = {0, 1, 2, 4 * GB - 1, 4 * GB, 4 * GB + 1, 5 * GB + 3, 300 * GB + 17}
    for b in BLOCK.values():
        s |= {b - 1, b, b + 1}
    return sorted(s)


def begin(ours, p):
    ctx = ctypes.c_void_p()
    ours.LizardF_createCompressionContext(ctypes.byref(ctx), 100)
    buf = ctypes.create_string_buffer(16)
    try:
        r = ours.LizardF_compressBegin(ctx, buf, 16, ctypes.byref(p))
    finally:
        ours.LizardF_freeCompressionContext(ctx)
    return r, buf.raw


PREF_SWEEP = [(bsid, mode, ck, cs, level) for bsid in range(9) for mode in (0, 1) for ck in (False, True) for cs in (0, 1)
              for level in (GPU_LEVEL, REFUSED_LEVEL)]


def test_plan_equals_this_librarys_bound_and_begin(shim, ours):
    """The header function against LizardF_compressFrameBound + LizardF_compressBegin of this library, and a plain statement
    of the block count and the staging bytes."""
    checked = {"ok": 0, "bound": 0, "other": 0}
    for bsid, mode, ck, cs, level in PREF_SWEEP:
        for n in sizes_to_check():
            p = one_shot(bsid, mode, ck, cs, n)
            p.compressionLevel = level
            bound = ours.LizardF_compressFrameBound(n, ctypes.byref(p))
            for cap in (bound - 1, bound, bound + 1):
                v, hdr, out = plan(shim, bsid, mode, ck, cs, level == GPU_LEVEL, n, cap)
                if cap < bound:
                    assert v == TOO_SMALL, (bsid, mode, ck, cs, level, n, cap, v)
                    checked["bound"] += 1
                    continue
                r, buf = begin(ours, p)
                if ours.LizardF_isError(r):
                    assert v == (1 << 64) - r and hdr == b"", (bsid, mode, ck, cs, level, n, v, r)
                    checked["other"] += 1
                    continue
                assert v == 0 and hdr == buf[:r], (bsid, mode, ck, cs, level, n, v, r, hdr, buf)
                bs = block_size(p.frameInfo.blockSizeID)
                nb = -(-n // bs)
                stage = (nb - 1) * bs + ((n - (nb - 1) * bs + 15) // 16) * 16 if nb else 0   # full blocks, the last rounded up
                assert out == [r, bs, nb, stage, int(ck)], (bsid, mode, ck, cs, n, out)
                checked["ok"] += 1
    assert min(checked.values()) > 100, checked


def test_plan_quirks(shim, ours):
    """The quirks as the host call has them: an out-of-range block size ID that becomes a valid one for a small input,
    blockSizeID 0, a content-size flag on an empty input, linked preferences on a single-block input."""
    v, hdr, out = plan(shim, 8, 1, False, 0, True, 1000, 1 << 20)            # ID 8 -> 128 KiB for 1000 bytes
    assert v == 0 and hdr[5] == 1 << 4 and out[1] == 128 * KB
    v, hdr, out = plan(shim, 8, 1, False, 0, True, 300 * MB, 1 << 40)        # ID 8 stays 8 above 256 MiB
    assert v == 2
    v, hdr, out = plan(shim, 0, 1, False, 0, True, 5, 100)                   # ID 0 is written as 1
    assert v == 0 and hdr[5] == 1 << 4
    v, hdr, out = plan(shim, 4, 1, False, 1, True, 0, 100)                   # no content size on an empty input
    assert v == 0 and len(hdr) == 7 and not hdr[4] & 8
    v, hdr, out = plan(shim, 1, 0, False, 0, True, 128 * KB, 1 << 20)        # linked, one block: independent
    assert v == 0 and hdr[4] & 0x20
    v, hdr, out = plan(shim, 1, 0, False, 0, True, 128 * KB + 1, 1 << 20)    # linked, two blocks: refused
    assert v == 3


def test_header_equals_reference_frames(shim, ours, ref):
    """Where the reference's LizardF_compressFrame writes a frame, its header bytes are the plan's, and it also refuses a
    capacity below the bound."""
    compared = 0
    for bsid, mode, ck, cs, level in PREF_SWEEP:
        if level != GPU_LEVEL:
            continue
        for n in (0, 1, 2, 128 * KB - 1, 128 * KB, 128 * KB + 1, 256 * KB + 1, MB + 1):
            data = lz.datagen(n, 50, n + bsid)[:n] if n else b""
            p = lz.make_prefs(GPU_LEVEL, bsid, mode == 1, ck, n if cs else 0)
            bound = ref.LizardF_compressFrameBound(n, ctypes.byref(p))
            assert bound == ours.LizardF_compressFrameBound(n, ctypes.byref(p)), (bsid, mode, ck, cs, n)
            for cap in (bound - 1, bound):
                v, hdr, _ = plan(shim, bsid, mode, ck, n if cs else 0, True, n, cap)
                dst = ctypes.create_string_buffer(cap + 64)                # it writes past a small capacity
                r = ref.LizardF_compressFrame(dst, cap, data, n, ctypes.byref(p))
                if cap < bound:
                    assert v == TOO_SMALL and ref.LizardF_isError(r) and (1 << 64) - r == TOO_SMALL
                elif v == 0 and not ref.LizardF_isError(r):
                    assert dst.raw[:len(hdr)] == hdr, (bsid, mode, ck, cs, n)
                    compared += 1
    assert compared > 150, compared


# ---- admission -----------------------------------------------------------------------------------------------------------------
def demands(sizes, caps, bsid):
    """(blocks, staging bytes) each frame asks for, stated plainly: nothing for a frame below its bound or an empty one."""
    out = []
    for n, c in zip(sizes, caps):
        p = one_shot(bsid, 1, True, 0, n)
        bs = block_size(p.frameInfo.blockSizeID)
        bound = frame_bound(n, bs)
        if c < bound or n == 0:
            out.append((0, 0))
            continue
        nb = -(-n // bs)
        out.append((nb, (nb - 1) * bs + ((n - (nb - 1) * bs + 15) // 16) * 16))
    return out


def frame_bound(n, bs):
    """LizardF_compressFrameBound with autoFlush and the content checksum."""
    nb = n // bs + 1
    return 15 + 4 * nb + bs * (nb - 1) + n % bs + 4 + 4


def admit(shim, sizes, caps, bsid, max_blocks, stage):
    n = len(sizes)
    s = np.array(sizes, dtype=np.uint64); c = np.array(caps, dtype=np.uint64)
    adm = np.zeros(n, dtype=np.uint32); first = np.zeros(n, dtype=np.uint64); sbase = np.zeros(n, dtype=np.uint64)
    shim.lzb_host_frame_compress_admit(n, s.ctypes.data, c.ctypes.data, bsid, 1, 1, 0, 1, max_blocks, stage, adm.ctypes.data,
                                       first.ctypes.data, sbase.ctypes.data)
    return [bool(a) for a in adm], [int(x) for x in first], [int(x) for x in sbase]


def prefix_rule(dem, max_blocks, stage):
    adm, first, sbase, cb, cs = [], [], [], 0, 0
    for b, s in dem:
        first.append(cb); sbase.append(cs)
        cb += b; cs += s
        adm.append(cb <= max_blocks and cs <= stage)
    return adm, first, sbase


def check(shim, sizes, caps, bsid, max_blocks, stage):
    got = admit(shim, sizes, caps, bsid, max_blocks, stage)
    want = prefix_rule(demands(sizes, caps, bsid), max_blocks, stage)
    assert got[0] == want[0], (max_blocks, stage)
    assert got[0] == sorted(got[0], reverse=True)
    for a, gf, gs, wf, ws in zip(got[0], got[1], got[2], want[1], want[2]):
        if a:
            assert (gf, gs) == (wf, ws)
    return got[0]


def _frames(rng, n, bsid):
    bs = BLOCK[bsid]
    sizes, caps = [], []
    for i in range(n):
        kind = i % 7
        size = 0 if kind == 3 else int(rng.integers(1, 4 * bs))
        cap = frame_bound(size, block_size(one_shot(bsid, 1, True, 0, size).frameInfo.blockSizeID))
        if kind == 5:
            cap -= 1                                                      # below the bound: takes nothing
        sizes.append(size); caps.append(cap)
    return sizes, caps


def test_admission_cuts_exactly(shim):
    rng = np.random.default_rng(7)
    for bsid in (1, 3):
        sizes, caps = _frames(rng, 40, bsid)
        dem = demands(sizes, caps, bsid)
        cb, cs = np.cumsum([b for b, _ in dem]), np.cumsum([s for _, s in dem])
        assert any(b == 0 for b, _ in dem[:10]) and any(b == 0 for b, _ in dem[-10:])
        for k in range(len(sizes)):
            adm = check(shim, sizes, caps, bsid, int(cb[k]), int(cs[-1]))
            assert adm[k]
            if dem[k][0]:
                assert not check(shim, sizes, caps, bsid, int(cb[k]) - 1, int(cs[-1]))[k]
            adm = check(shim, sizes, caps, bsid, int(cb[-1]), int(cs[k]))
            assert adm[k]
            if dem[k][1]:
                assert not check(shim, sizes, caps, bsid, int(cb[-1]), int(cs[k]) - 1)[k]
        assert check(shim, sizes, caps, bsid, 0, 0)[:1] == [dem[0] == (0, 0)]


def test_admission_random(shim):
    rng = np.random.default_rng(9)
    for trial in range(200):
        bsid = (1, 2, 4)[trial % 3]
        sizes, caps = _frames(rng, int(rng.integers(1, 50)), bsid)
        dem = demands(sizes, caps, bsid)
        tb, ts = sum(b for b, _ in dem), sum(s for _, s in dem)
        for mb, st in ((tb, ts), (int(rng.integers(0, tb + 2)), ts), (tb, int(rng.integers(0, ts + 2))), (0, 0)):
            check(shim, sizes, caps, bsid, mb, st)


def test_stage_clamp(shim):
    """stageBytes up to SIZE_MAX: at most maxBlocks blocks of the preferences' block size (256 MiB for an invalid ID), and the
    clamped bound admits the same frames as the caller's."""
    for bsid in range(10):
        top = BLOCK.get(1 if bsid == 0 else bsid, 256 * MB)
        for mb in (0, 1, 8192, (1 << 32) - 1):
            for stage in (0, 1, mb * top - 1, mb * top, mb * top + 1, SIZE_MAX - 64, SIZE_MAX):
                if stage < 0:
                    continue
                got = shim.lzb_host_frame_compress_stage_limit(mb, bsid, stage)
                assert got == min(stage, mb * top) and got <= 1 << 60, (bsid, mb, stage, got)
    rng = np.random.default_rng(13)
    for trial in range(50):
        sizes, caps = _frames(rng, 30, 1)
        dem = demands(sizes, caps, 1)
        mb = int(rng.integers(0, sum(b for b, _ in dem) + 2))
        assert check(shim, sizes, caps, 1, mb, SIZE_MAX) == prefix_rule(dem, mb, 1 << 62)[0]


# ---- resource figures of the new kernels -------------------------------------------------------------------------------------
# DESIGN.md 3.4c lists these figures
COMPRESS_ASYNC_KERNEL_LIMITS = {
    "lizard_frames_compress_tile_kernel": (32, 0),
    "lizard_frames_compress_plan_kernel": (32, 0),
    "lizard_frames_compress_blocks_kernel": (29, 0),
    "lizard_frames_compress_verdict_kernel": (10, 0),
}


def test_compress_async_kernel_resources():
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
            for k in COMPRESS_ASYNC_KERNEL_LIMITS:
                if re.search(r"\d" + k + r"[A-Z]", name):
                    found[k] = {a: int(b) for a, b in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    assert set(found) == set(COMPRESS_ASYNC_KERNEL_LIMITS), found
    for k, (reg, stack) in COMPRESS_ASYNC_KERNEL_LIMITS.items():
        r = found[k]
        assert r["REG"] <= reg and r["STACK"] <= stack and r["LOCAL"] == 0, (k, r)
