"""LizardB200_decompressFramesAsync (DESIGN.md 3.4b) on the CPU: the host build (lizard_b200/libhostshim.so, TEST-ONLY) of the
serial rules its kernels run.

- The planning (frame_plan_blocks / frame_admit_blocks / frame_admit_slots in the two steps the kernels take) admits the
  prefix a plain statement of the rule gives, on random block counts, slot sizes and bounds, exact fits and misses by one of
  both bounds, frames of no blocks and frames with a bad header.
- frame_settle_entries on the device-side layout (slots behind each other, one staged and one raw gather entry per block)
  gives the host loop's verdicts and bytes (lzb_host_frame_decode) on the frames test_frame_device_cpu.py builds.
- The new kernels' registers, stack and local memory, read with cuobjdump -res-usage."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from tests import refs
from tests.test_encode_resources_cpu import _cuobjdump
from tests.test_frame_device_cpu import _damaged, _ref_frames, host_frames, ref  # noqa: F401 (fixture)

U64 = ctypes.c_ulonglong


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    L.lzb_host_frame_async_plan.argtypes = [ctypes.c_uint, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint,
                                            U64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.lzb_host_frame_stage_limit.argtypes = [ctypes.c_uint, U64]
    L.lzb_host_frame_stage_limit.restype = U64
    L.lzb_host_frame_async_decode.argtypes = [ctypes.c_char_p, U64, ctypes.c_void_p, U64]
    L.lzb_host_frame_async_decode.restype = U64
    L.lzb_host_frame_decode.argtypes = [ctypes.c_char_p, U64, ctypes.c_void_p, U64, ctypes.POINTER(ctypes.c_uint)]
    L.lzb_host_frame_decode.restype = U64
    return L


# ---- planning -------------------------------------------------------------------------------------------------------------
def plan(shim, blocks, slots, ok, max_blocks, stage):
    n = len(blocks)
    b = np.array(blocks, dtype=np.uint64); s = np.array(slots, dtype=np.uint64); o = np.array(ok, dtype=np.uint32)
    adm = np.zeros(n, dtype=np.uint32); base = np.zeros(n, dtype=np.uint64); slot = np.zeros(n, dtype=np.uint64)
    shim.lzb_host_frame_async_plan(n, b.ctypes.data, s.ctypes.data, o.ctypes.data, max_blocks, stage, adm.ctypes.data,
                                   base.ctypes.data, slot.ctypes.data)
    return [bool(a) for a in adm], [int(x) for x in base], [int(x) for x in slot]


def prefix_rule(blocks, slots, ok, max_blocks, stage):
    """Frame i is admitted while the frames 0..i take at most max_blocks blocks and stage bytes of slots; a bad header takes
    nothing.  Returns the admission and, for admitted frames, the block and slot bases."""
    adm, base, slot, cb, cs = [], [], [], 0, 0
    for b, s, o in zip(blocks, slots, ok):
        b, s = (b, s) if o else (0, 0)
        base.append(cb); slot.append(cs)
        cb += b; cs += s
        adm.append(cb <= max_blocks and cs <= stage)
    return adm, base, slot


def check_plan(shim, blocks, slots, ok, max_blocks, stage):
    got = plan(shim, blocks, slots, ok, max_blocks, stage)
    want = prefix_rule(blocks, slots, ok, max_blocks, stage)
    assert got[0] == want[0], (blocks, slots, ok, max_blocks, stage)
    assert got[0] == sorted(got[0], reverse=True)                    # a prefix
    for a, gb, gs, wb, ws in zip(got[0], got[1], got[2], want[1], want[2]):
        if a:
            assert (gb, gs) == (wb, ws)
    return got[0]


def test_plan_matches_the_prefix_rule(shim):
    rng = np.random.default_rng(3)
    for trial in range(400):
        n = int(rng.integers(1, 60))
        blocks = [int(x) for x in rng.integers(0, 6, n)]
        mb = [128 << 10, 4 << 20, 256 << 20][trial % 3]
        slots = [int(rng.integers(0, b + 1)) * mb for b in blocks]     # some blocks raw
        ok = [int(x) for x in rng.random(n) > 0.15]
        tb = sum(b for b, o in zip(blocks, ok) if o)
        ts = sum(s for s, o in zip(slots, ok) if o)
        for max_blocks, stage in ((tb, ts), (int(rng.integers(0, tb + 2)), ts), (tb, int(rng.integers(0, ts + 2))),
                                  (int(rng.integers(0, tb + 2)), int(rng.integers(0, ts + 2))), (0, 0)):
            check_plan(shim, blocks, slots, ok, max_blocks, stage)


def test_plan_exact_fit_and_one_over(shim):
    blocks = [3, 0, 2, 5, 0, 1, 4, 2]
    slots = [3 << 17, 0, 1 << 17, 5 << 17, 0, 0, 4 << 17, 2 << 17]
    ok = [1, 1, 0, 1, 1, 1, 0, 1]                                      # frames 2 and 6: bad headers
    cb = np.cumsum([b * o for b, o in zip(blocks, ok)])
    cs = np.cumsum([s * o for s, o in zip(slots, ok)])
    for k in range(len(blocks)):
        adm = check_plan(shim, blocks, slots, ok, int(cb[k]), int(cs[-1]))          # exact fit of the blocks
        assert adm[k] and (k + 1 == len(blocks) or cb[k + 1] > cb[k] or adm[k + 1])
        if cb[k] > 0:
            adm = check_plan(shim, blocks, slots, ok, int(cb[k]) - 1, int(cs[-1]))  # one block short
            assert not adm[k]
        adm = check_plan(shim, blocks, slots, ok, int(cb[-1]), int(cs[k]))          # exact fit of the slots
        assert adm[k]
        if cs[k] > 0:
            adm = check_plan(shim, blocks, slots, ok, int(cb[-1]), int(cs[k]) - 1)  # one byte short
            assert not adm[k]
    assert check_plan(shim, [0, 0, 0], [0, 0, 0], [1, 0, 1], 0, 0) == [True] * 3    # frames of no blocks need nothing


def test_stage_bound_never_wraps(shim):
    """stageBytes up to SIZE_MAX: the arena is sized for at most maxBlocks slots of 256 MiB (no room for `+ 64` to wrap), and
    the clamped bound admits the same frames as the caller's."""
    most = 256 << 20
    size_max = (1 << 64) - 1
    for mb in (0, 1, 7, 8192, (1 << 32) - 1):
        for stage in (0, 1, mb * most - 1, mb * most, mb * most + 1, size_max - 64, size_max - 63, size_max):
            if stage < 0:
                continue
            got = shim.lzb_host_frame_stage_limit(mb, stage)
            assert got == min(stage, mb * most) and got <= (1 << 60), (mb, stage, got)
    rng = np.random.default_rng(11)
    for trial in range(100):
        n = int(rng.integers(1, 40))
        blocks = [int(x) for x in rng.integers(0, 4, n)]
        slots = [int(rng.integers(0, b + 1)) * (256 << 20) for b in blocks]
        ok = [1] * n
        mbk = int(rng.integers(0, sum(blocks) + 2))
        for stage in (size_max, size_max - 63):                       # "no staging bound"
            assert check_plan(shim, blocks, slots, ok, mbk, stage) == prefix_rule(blocks, slots, ok, mbk, 1 << 62)[0]


# ---- settling on the device-side layout ---------------------------------------------------------------------------------------
def async_frames(shim, frame: bytes, cap: int):
    dst = ctypes.create_string_buffer(b"\xA5" * (cap + 64), cap + 64)
    r = shim.lzb_host_frame_async_decode(frame, len(frame), dst, cap)
    assert dst.raw[cap:] == b"\xA5" * 64, "wrote behind the capacity"
    return r, dst.raw[:r] if r < (1 << 63) else b""


def test_settle_entries_reference_frames(ref, shim):
    for name, frame, n in _ref_frames(ref):
        for cap in sorted({n, n + 1, n + 1000, max(n - 1, 0), n // 2, 0, 3 * (128 << 10) + 11}):
            assert async_frames(shim, frame, cap) == host_frames(shim, frame, cap), (name, cap)


def test_settle_entries_skippable_and_damaged(ref, shim):
    body = b"skip me" * 10
    sk = (0x184D2A53).to_bytes(4, "little") + len(body).to_bytes(4, "little") + body
    for frame in (sk, sk[:-1], sk + b"x", sk[:7], sk[:8], sk[:3]):
        for cap in (0, 100):
            assert async_frames(shim, frame, cap) == host_frames(shim, frame, cap), (len(frame), cap)
    for name, frame, cap, _ in _damaged(ref):                        # linked, truncated, trailing, above the maximum, ...
        got, want = async_frames(shim, frame, cap), host_frames(shim, frame, cap)
        assert got[0] == want[0], (name, cap, got[0], want[0])
        assert got[1] == want[1], name


# ---- resource figures of the new kernels --------------------------------------------------------------------------------
# DESIGN.md 3.4b lists these figures
ASYNC_KERNEL_LIMITS = {
    "lizard_frames_async_tile_kernel": (32, 0),
    "lizard_frames_async_plan_kernel": (32, 0),
    "lizard_frames_async_settle_kernel": (56, 0),
    "lizard_frames_async_hash_kernel": (72, 0),
    "lizard_frames_async_verdict_kernel": (9, 0),
}


def test_async_kernel_resources():
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
            for k in ASYNC_KERNEL_LIMITS:
                if re.search(r"\d" + k + r"[A-Z]", name):
                    found[k] = {a: int(b) for a, b in re.findall(r"(REG|STACK|LOCAL|SHARED):(\d+)", line)}
            name = None
    assert set(found) == set(ASYNC_KERNEL_LIMITS), found
    for k, (reg, stack) in ASYNC_KERNEL_LIMITS.items():
        r = found[k]
        assert r["REG"] <= reg and r["STACK"] <= stack and r["LOCAL"] == 0, (k, r)
