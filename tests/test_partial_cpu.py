"""Lizard_decompress_safe_partial through the device decoder's code on the CPU: the one-lane host build and the 32-lane warp
emulator of the partial kernel (lizard_b200/libhostshim.so, TEST-ONLY) against the compiled reference.  Return codes must
always be equal; the bytes in front of the returned size must be equal whenever the stream obeys the min-offset rule (below
it the reference's own output depends on stale memory).  Bytes behind the returned size are unspecified, but nothing may be
written behind the capacity.

The reference stops in three places (lib/lizard_decompress.c, lib/lizard_decompress_lz4.h, lib/lizard_decompress_liz.h):
after a token's literals or after its match (fastLZ4 codewords, :82 / :144), in front of a token (LIZv1, :55), and after
an inner block (:175 raw, :249 compressed).  The token loops measure the target from the start of their inner block, the
unit loop from the start of the unit.  Also checked here: the full-decode kernel instances keep the register and stack
figures they had before the partial kernel was added, and the partial kernel is an instance of its own."""
import ctypes
import functools
import os
import random
import re
import subprocess

import pytest

import lizard_b200 as lz
from tests import corpus, refs
from tests.test_encode_resources_cpu import _cuobjdump

BS = lz.BLOCK_SIZE
HOST, EMU = "lzb_host_decompress_partial", "lzb_emu_decompress_partial"
GUARD = 64


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    L.Lizard_decompress_safe_partial.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return L


@pytest.fixture(scope="module")
def shim():
    p = os.path.join(refs.ROOT, "lizard_b200", "libhostshim.so")
    if not os.path.exists(p):
        pytest.skip("libhostshim.so not built")
    L = ctypes.CDLL(p)
    for f in (HOST, EMU):
        getattr(L, f).argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
    L.lzb_host_decompress.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    return L


def ref_partial(ref, comp, target, cap):
    # room behind the capacity: the reference's wild copies write up to 16 bytes past its cursor, and it does not charge a
    # raw inner block against the capacity (DESIGN.md 3.5)
    dst = ctypes.create_string_buffer(2 * max(cap, 1) + 64)
    r = ref.Lizard_decompress_safe_partial(comp, dst, len(comp), target, cap)
    return r, dst.raw[:max(r, 0)]


def dev_partial(shim, fn, comp, target, cap):
    dst = ctypes.create_string_buffer(b"\xA5" * (cap + GUARD), cap + GUARD)
    r = getattr(shim, fn)(comp, len(comp), dst, target, cap)
    assert dst.raw[cap:] == b"\xA5" * GUARD, (fn, target, cap, "wrote behind the capacity")
    return r, dst.raw[:max(r, 0)]


@functools.lru_cache(maxsize=None)
def _obeys(comp, size):
    return refs.stream_obeys_min_offset(comp, size)


def check(ref, shim, comp, size, targets, cap=None, fns=(HOST, EMU)):
    """Every target through every function: the reference's return code, its bytes where they are defined.  `size` = the
    stream's decoded size (for the min-offset rule).  Returns the reference's results."""
    cap = size if cap is None else cap
    out = []
    for t in targets:
        rr, ro = ref_partial(ref, comp, t, cap)
        for fn in fns:
            r, o = dev_partial(shim, fn, comp, t, cap)
            assert r == rr, (fn, len(comp), size, cap, t, r, rr)
            if rr > 0 and _obeys(comp, size):
                assert o == ro, (fn, len(comp), size, cap, t)
        out.append(rr)
    return out


@functools.lru_cache(maxsize=None)
def _level_inputs(level):
    """Small units of every kind: datagen, a codeword-threshold block, periodic data, a Huffman-hostile block, and a unit of
    two inner blocks."""
    fams = corpus.corpus()
    thr = fams["threshold"][5 if corpus.is_lizv1(level) else 0]
    return [lz.datagen(20000, 50, level), thr[:24000], fams["periodic"][3], fams["periodic"][-2], fams["hostile"][0][:8192],
            fams["hostile"][3][:5000], lz.datagen(BS + 5000, 60, level)]


@pytest.mark.parametrize("level", range(10, 50))
def test_every_level_matches_reference(ref, shim, level):
    """Every level 10-49: the reference's streams of datagen and corpus units at targets -1, 0, 1, random ones, around the
    decoded size and far beyond it.  The emulator takes the small units at a subset of the targets."""
    rnd = random.Random(level)
    for u in _level_inputs(level):
        comp = refs.ref_compress(ref, u, level)
        n = len(u)
        targets = [-1, 0, 1, rnd.randrange(2, n), rnd.randrange(2, n), n // 2, n - 1, n, n + 1, 1 << 30]
        check(ref, shim, comp, n, targets, fns=(HOST,))
        if n < BS:
            check(ref, shim, comp, n, [-1, 0, 1, rnd.randrange(2, n), n], fns=(EMU,))


def _sweep_boundaries(ref, comp, n):
    """Every target from -1 to n + 1 through the reference: the set of places where it stops."""
    return sorted({ref_partial(ref, comp, t, n)[0] for t in range(-1, n + 2)})


@pytest.mark.parametrize("level", [10, 30, 20, 21, 41])
def test_every_token_boundary(ref, shim, level):
    """A block of ~100 tokens: the one-lane build at every target from -1 to n + 1, the emulator at every place the reference
    stops and one byte either side (after a token's literals or in the middle of its match for fastLZ4, at a token's start
    for LIZv1).  Exits fall on every lane of a 32-token batch, and behind a failed check nowhere."""
    data = lz.datagen(6000, 50, 3) + corpus.periodic_units()[0][:1500]
    comp = refs.ref_compress(ref, data, level)
    n = len(data)
    check(ref, shim, comp, n, range(-1, n + 2), fns=(HOST,))
    stops = _sweep_boundaries(ref, comp, n)
    assert len(stops) > 40, (level, len(stops))
    targets = sorted({b + d for b in stops for d in (-1, 0, 1)})
    check(ref, shim, comp, n, targets, fns=(EMU,))
    last = max(b for b in stops if b < n)
    if corpus.is_lizv1(level):
        # in front of the last token: once it ran, the flags are out and the block's last literals follow
        assert ref_partial(ref, comp, last + 1, n)[0] == n
    else:
        # the stop after the last token's match: the block's last literals are not copied
        assert ref_partial(ref, comp, last, n)[0] == last < n


@pytest.mark.parametrize("level", [10, 30])
def test_lz4_block_ending_at_or_past_the_target_keeps_its_last_literals_out(ref, shim, level):
    """fastLZ4 blocks with literal tails of many lengths: a target at or inside the last token's match stops there, without
    the block's last literals (lizard_decompress_lz4.h:144 returns before :148)."""
    rnd = random.Random(level)
    seen = 0
    for k in range(12):
        data = lz.datagen(3000 + 37 * k, 40 + 3 * k, k) + bytes(rnd.randrange(256) for _ in range(k * 7))
        comp = refs.ref_compress(ref, data, level)
        n = len(data)
        ends = [ref_partial(ref, comp, t, n)[0] for t in range(n - 200, n + 1)]
        tail = [t for t, r in zip(range(n - 200, n + 1), ends) if t <= r < n]
        if tail:
            seen += 1
            check(ref, shim, comp, n, [tail[-1] - 1, tail[-1], tail[-1] + 1, n])
    assert seen >= 6, seen


@pytest.mark.parametrize("level", [10, 21, 41])
def test_inner_block_boundaries_and_the_block_relative_target(ref, shim, level):
    """A unit of four inner blocks.  The token loop of block k stops at its own start + target, the unit loop at the unit's
    start + target: a target between blocks decodes the block it falls in whole, and 200000 returns 262144."""
    data = lz.datagen(3 * BS + 7000, 50, level)
    comp = refs.ref_compress(ref, data, level)
    n = len(data)
    targets = [BS - 1, BS, BS + 1, 200000, 2 * BS - 1, 2 * BS, 2 * BS + 1, 300000, 3 * BS, 3 * BS + 1, n - 1, n, n + 1, 1, 4000]
    got = check(ref, shim, comp, n, targets, fns=(HOST,))
    assert got[targets.index(200000)] == 2 * BS
    assert got[targets.index(BS + 1)] == 2 * BS and got[targets.index(2 * BS + 1)] == 3 * BS
    check(ref, shim, comp, n, [BS - 1, BS + 1, 200000, 4000], fns=(EMU,))


@pytest.mark.parametrize("level", [10, 21, 41])
def test_raw_inner_block_before_a_compressed_one(ref, shim, level):
    """An incompressible first inner block is stored raw; it is copied whole and then compared with the target (:175), so
    even target 0 returns 131072."""
    import numpy as np
    data = np.random.default_rng(level).integers(0, 256, BS, dtype=np.uint8).tobytes() + lz.datagen(40000, 50, level)
    comp = refs.ref_compress(ref, data, level)
    assert comp[1] == 0x80
    n = len(data)
    targets = [-1, 0, 1, 65536, BS - 1, BS, BS + 1, BS + 20000, n - 1, n, n + 1]
    got = check(ref, shim, comp, n, targets, fns=(HOST,))
    assert got[:3] == [BS, BS, BS]
    check(ref, shim, comp, n, [0, BS, BS + 1, BS + 20000], fns=(EMU,))


def test_target_at_or_above_the_decoded_size_is_decompress_safe(ref, shim):
    for level in (10, 20, 30, 41, 17, 45):
        for data in (lz.datagen(9000, 50, level), lz.datagen(BS + 333, 30, level), b"", b"x" * 40):
            comp = refs.ref_compress(ref, data, level)
            n = len(data)
            full = refs.ref_decompress(ref, comp, n)
            for t in (n, n + 1, 2 ** 31 - 1):
                assert ref_partial(ref, comp, t, n) == full
            check(ref, shim, comp, n, (n, n + 1, 2 ** 31 - 1), fns=(HOST,) if n > BS else (HOST, EMU))
            dst = ctypes.create_string_buffer(max(n, 1) + 64)
            assert shim.lzb_host_decompress(comp, len(comp), dst, n) == full[0]


@pytest.mark.parametrize("level", [10, 21, 41, 30])
def test_capacity_too_small(ref, shim, level):
    """Capacities below the decoded size: the checks in front of the stopping point fail exactly where the reference's do,
    the ones behind it never run."""
    data = lz.datagen(20000, 50, level)
    comp = refs.ref_compress(ref, data, level)
    n = len(data)
    for cap in (0, 1, 15, 16, 17, 100, 4096, n // 2, n - 1):
        check(ref, shim, comp, n, [-1, 0, 1, 50, n // 4, n // 2, n - 20, n], cap=cap, fns=(HOST,))
        check(ref, shim, comp, n, [0, 50, n // 4, n], cap=cap, fns=(EMU,))


def _le24(b, at):
    return b[at] | (b[at + 1] << 8) | (b[at + 2] << 16)


def _token_streams(comp):
    """(start, end) in `comp` of the offset and flags streams of every compressed inner block: damage there breaks the token
    loop (damage in the literals mostly changes bytes only)."""
    out, ip = [], 1
    while ip < len(comp):
        hdr = comp[ip]
        ip += 1
        if hdr == 0x80:
            ip += 3 + _le24(comp, ip)
            continue
        ip += 3 + _le24(comp, ip)                               # lengths stream
        start = ip
        for flag in (4, 8, 2, 1):                              # offset16, offset24, flags, literals; Huffman-coded when set
            if flag == 1:
                out.append((start, ip))
            ip += 6 + _le24(comp, ip + 3) if hdr & flag else 3 + _le24(comp, ip)
    return out


def _damage(rnd, comp, lo, hi):
    b = bytearray(comp)
    for _ in range(rnd.choice([1, 1, 3])):
        at = rnd.randrange(lo, hi)
        b[at] ^= (1 << rnd.randrange(8)) if rnd.random() < 0.5 else rnd.randrange(1, 256)
    return bytes(b)


@pytest.mark.parametrize("level", [10, 20, 21, 30, 41])
def test_damage_in_front_of_and_behind_the_stopping_point(ref, shim, level):
    """Damaged streams: damage in front of the stopping point gives the reference's error, damage behind it is never read
    and the call succeeds, as in the reference.  A unit of two inner blocks, damaged in the offset and flags streams of one
    of them, decoded to targets in both blocks: both outcomes must occur."""
    rnd = random.Random(900 + level)
    data = lz.datagen(BS + 30000, 50, level)
    comp = refs.ref_compress(ref, data, level)
    n = len(data)
    blocks = _token_streams(comp)
    assert len(blocks) == 2, blocks
    accepted_behind = failed_in_front = 0
    for k in range(40):
        lo, hi = blocks[k % 2]
        bad = _damage(rnd, comp, lo, hi)
        full = refs.ref_decompress(ref, bad, n)[0]
        targets = [rnd.randrange(-1, 3000), rnd.randrange(0, BS - 100), rnd.randrange(BS, n + 10)]
        got = check(ref, shim, bad, n, targets, fns=(HOST,))
        check(ref, shim, bad, n, targets[:1], fns=(EMU,))
        accepted_behind += sum(1 for r in got if r > 0) if full < 0 else 0
        failed_in_front += sum(1 for r in got if r < 0)
    assert accepted_behind > 0 and failed_in_front > 0, (accepted_behind, failed_in_front)


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not _no_gpu(), reason="checks the behaviour when no CUDA device is present")
def test_partial_calls_fail_without_a_gpu_instead_of_falling_back():
    L = lz.lib()
    unit = b"\x0a\x80\x01\x00\x00a"                            # level 10, one raw inner block of one byte
    assert lz.decompress_partial(unit, 1, 64)[0] < 0
    assert lz.decompress_partial(b"", 1, 64) == (0, b"")        # compressedSize < 1 returns 0 before anything is read
    with pytest.raises(lz.LizardB200Error):
        lz.decompress_partial_batch([unit], [1], [64])
    assert L.LizardB200_lastError()
    one = ctypes.c_int(1)
    assert L.LizardB200_decompress_partial_device(None, None, None, None, None, None, ctypes.byref(one), ctypes.byref(one),
                                                  1, None) < 0


# ---------------------------------------------------------------------------------------------------------------------
# compiled kernels
# ---------------------------------------------------------------------------------------------------------------------
# the first-generation full-decode instances (schedule V = 0..3) as they were before the partial kernel existed: adding it
# must not change their code.  (sm_90a, CUDA 12.9)
FULL_DECODE = {0: {"REG": 64, "STACK": 528}, 1: {"REG": 64, "STACK": 672}, 2: {"REG": 64, "STACK": 544}, 3: {"REG": 64, "STACK": 688}}


def _decode_instances():
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
            f = re.search(r"lizard_decode_units_kernelILi(\d+)E", name)
            key = int(f.group(1)) if f else ("partial" if "lizard_decode_partial_units_kernel" in name else None)
            if key is not None:
                found[key] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            name = None
    return found


def test_full_decode_instances_keep_their_resources():
    inst = _decode_instances()
    for v, want in FULL_DECODE.items():
        assert {k: inst[v][k] for k in want} == want, (v, inst[v])


def test_partial_decode_is_its_own_kernel_within_the_token_kernels_registers():
    inst = _decode_instances()
    assert "partial" in inst, sorted(inst, key=str)
    assert inst["partial"]["REG"] <= 64 and inst["partial"]["LOCAL"] == 0, inst["partial"]
