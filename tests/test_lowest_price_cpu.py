"""The lowestPrice encoder (levels 23-25 and their Huffman twins 43-45) without a GPU: the one-lane host build and the 32-lane
warp emulator (all three lane orders) of encode_lp.cuh must write the bytes of the reference built with -DLIZARD_RESET_MEM.
Also: the rare paths are reached (short repeat matches, 24-bit offsets, both outcomes of Lizard_more_profitable, the price
scan's terminating branch), the levels stay refused where they always were, and the new kernel's resources are pinned."""
import ctypes
import os
import random
import re
import subprocess

import numpy as np
import pytest

import lizard_b200 as lz
from tests import refs
from tests.corpus import corpus
from tests.test_encode_resources_cpu import LIB, _cuobjdump
from tests.test_gpu_encode import _cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = [23, 24, 25, 43, 44, 45]
BS = lz.BLOCK_SIZE
SHORT_REP, FAR_OFFSET, MORE_PROFITABLE_YES, MORE_PROFITABLE_NO, SCAN_ELSE, SEQUENCES = range(6)   # csrc/encode_lp.cuh


@pytest.fixture(scope="module")
def ref():
    L = refs.ref_parity()
    if L is None:
        pytest.skip("oracle/_ref not built")
    return L


@pytest.fixture(scope="module")
def shim():
    L = ctypes.CDLL(os.path.join(ROOT, "lizard_b200", "libhostshim.so"))
    for f in ("lzb_host_compress", "lzb_emu_compress"):
        getattr(L, f).argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
    L.lzb_emu_lane_order.argtypes = [ctypes.c_int]
    L.lzb_lp_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    return L


def _run(fn, data, level, cap):
    dst = ctypes.create_string_buffer(max(cap, 1) + 64)
    n = fn(data, len(data), dst, cap, level)
    return dst.raw[:n]


def _stats(shim):
    out = (ctypes.c_ulonglong * 6)()
    shim.lzb_lp_stats(out, 1)
    return list(out)


def _same(shim, ref, data, level, cap=None, emu=False):
    cap = ref.Lizard_compressBound(len(data)) if cap is None else cap
    want = refs.ref_compress(ref, data, level, cap)
    got = _run(shim.lzb_host_compress, data, level, cap)
    assert got == want, ("host", level, len(data), cap, len(got), len(want))
    if emu:
        for order in (0, 1, 2):
            shim.lzb_emu_lane_order(order)
            got = _run(shim.lzb_emu_compress, data, level, cap)
            assert got == want, ("emu", order, level, len(data), cap, len(got), len(want))
        shim.lzb_emu_lane_order(0)
    return want


@pytest.mark.parametrize("level", LEVELS)
def test_corpus_and_datagen(ref, shim, level):
    units = [u for fam in corpus().values() for u in fam]
    for p in (0, 10, 50, 90, 100):
        units.append(lz.datagen(BS, p, p + level))
    for i, u in enumerate(units):
        _same(shim, ref, u, level, emu=i in (0, len(units) // 2, len(units) - 3))


@pytest.mark.parametrize("level", LEVELS)
def test_edge_sizes_and_capacities(ref, shim, level):
    rnd = random.Random(level)
    for c in _cases():
        want = _same(shim, ref, c, level)
        bound = ref.Lizard_compressBound(len(c))
        for cap in {bound, len(want), max(len(want) - 1, 1), max(len(want) // 2, 1)}:      # cap 0: the reference writes past it
            _same(shim, ref, c, level, cap, emu=len(c) in (1000, 4096) and rnd.random() < 0.3)


@pytest.mark.parametrize("level", LEVELS)
def test_units_of_several_inner_blocks(ref, shim, level):
    _same(shim, ref, lz.datagen(300000, 50, level), level)
    _same(shim, ref, lz.datagen(BS + 9000, 50, level), level, emu=level in (25, 45))
    _same(shim, ref, lz.datagen(1 << 20, 70, level), level)


@pytest.mark.parametrize("level", [25, 45])
def test_unit_beyond_the_window(ref, shim, level):
    """More than 4 MiB: matches reach 2^22 - 1 back, the chain wraps at 2^22 and the window cuts candidates off."""
    head = lz.datagen(3 << 20, 30, 9)
    data = head + lz.datagen(1 << 20, 60, 10) + head[:1 << 20] + head[1 << 20:(1 << 20) + 500000]
    _same(shim, ref, data, level)


def test_rare_paths_are_reached(ref, shim):
    _stats(shim)
    rng = np.random.default_rng(5)
    far = bytearray(lz.datagen(3 << 19, 40, 1))
    far[1 << 20:] = bytes(far[:len(far) - (1 << 20)])         # repeats 1 MiB back: 24-bit offsets
    units = [bytes(far)]
    for p in (20, 50, 80):
        units.append(lz.datagen(BS, p, 7 * p))
    # short repeats: a period-8 pattern broken by random bytes, so that runs of 2-3 bytes at the last offset appear
    a = bytearray((b"abcdefgh" * (BS // 8)))
    for i in rng.integers(0, BS, BS // 6):
        a[i] = int(rng.integers(0, 256))
    units.append(bytes(a))
    for level in (25, 45):
        for u in units:
            _same(shim, ref, u, level)
    s = _stats(shim)
    assert s[SHORT_REP] > 0 and s[FAR_OFFSET] > 0, s
    assert s[MORE_PROFITABLE_YES] > 0 and s[MORE_PROFITABLE_NO] > 0 and s[SCAN_ELSE] > 0, s


def _far_copies(seed, n=3 << 20):
    """Runs of 16-120 bytes copied from 2^16 .. 2^22 - 1 bytes back, some with one byte changed, between short random gaps:
    candidates at far offsets of different bit lengths compete, where the price's offset term depends on the Huffman flag."""
    rng = np.random.default_rng(seed)
    out = bytearray(lz.datagen(1 << 20, 20, seed))
    while len(out) < n:
        k = int(rng.integers(16, 120))
        at = len(out) - int(rng.integers(1 << 16, min(len(out), 1 << 22)))
        seg = bytearray(out[at:at + k])
        if rng.random() < 0.5:
            seg[int(rng.integers(0, k))] ^= 0x5A
        out += seg + bytes(rng.integers(0, 256, int(rng.integers(0, 6)), dtype=np.uint8))
    return bytes(out[:n])


def test_huffman_flag_changes_the_parse(ref, shim):
    """At 43-45 the price's offset and token terms differ (:284-290), so the parse itself differs from 23-25, beyond the
    entropy stage: on far-offset input the parser's own counts (sequences, 24-bit offsets, more_profitable outcomes; taken
    before any stream is built) differ between the twins, and both outputs still match the reference byte for byte."""
    data = _far_copies(1)
    for plain_level in (24, 25):
        _stats(shim)
        _same(shim, ref, data, plain_level)
        plain = _stats(shim)
        _same(shim, ref, data, plain_level + 20)
        huf = _stats(shim)
        assert plain[FAR_OFFSET] > 0 and plain[SEQUENCES] > 0
        assert plain != huf, (plain_level, plain, huf)


def test_level_12_stays_unsupported(shim):
    data = lz.datagen(5000, 50, 1)
    assert _run(shim.lzb_host_compress, data, 12, 10000) == b""


def test_kernel_resources():
    """lizard_encode_lowest_price_kernel at 128 threads under __maxnreg__(96): exactly 96 registers (5 CTAs per SM) and a
    496-byte frame (the entropy stage it inlines: ptxas reports 76 bytes of spill stores there), no local memory.  A change
    in either figure should be looked at before it is measured."""
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run([exe, "-res-usage", LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            found[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            name = None
    k = [n for n in found if "lizard_encode_lowest_price_kernel" in n]
    assert len(k) == 1 and not re.search(r"lizard_encode_units_kernelILi\d+E", k[0])
    assert found[k[0]] == {"REG": 96, "STACK": 496, "LOCAL": 0}, found[k[0]]
